// regex_dfa.cpp — the host half of -E searches: rebuilds the regular expression krep compiled (krep.c:2081-2145,
// 2539-2600), parses it as a glibc POSIX ERE in the C locale and compiles it into a LINE automaton: a DFA that reads
// one line (the bytes between two '\n') and tells whether the regex can match somewhere in it.
//
// The automaton is a filter, not a matcher.  It may say "yes" for a line glibc would not match (its answer is
// widened wherever modelling glibc exactly would take effort: \b \B \< \> become empty; an -i bracket expression whose
// parsed set is not closed under case still marks the plan widened, though its bytes are glibc's own), never "no" for a
// line glibc matches.  Positions, leftmost-longest choice, -w, -c and -m all come from glibc's regexec on the caller's
// own regex_t, run on the flagged lines only (replay_regex).
// Anything the parser does not know is refused, and a refused pattern stays on the host's regex_search.
//
// Under REG_NEWLINE (krep always sets it) no match contains a '\n' as long as no character set of the pattern contains
// one: '.' and non-matching lists exclude it, but \s, \W, [[:space:]] and [[:cntrl:]] do not — those are refused.
#include <algorithm>
#include <bitset>
#include <climits>
#include <cstdlib>
#include <cstring>
#include <map>
#include <regex.h>
#include <string>
#include <vector>
#include "common.h"

namespace kb {

namespace {

using CharSet = std::bitset<256>;

struct Ast
{
    enum Kind { EMPTY, SET, CAT, ALT, REP, BOL, EOL } kind = EMPTY;
    CharSet set;                 // SET
    std::vector<int> kids;       // CAT / ALT / REP (one kid)
    int min = 0, max = 0;        // REP; max < 0 = unbounded
};

struct Parser
{
    const std::string &s;
    size_t i = 0;
    bool icase;
    bool widened = false;
    std::string why; // non-empty once the pattern is refused
    std::vector<Ast> nodes;

    Parser(const std::string &src, bool ic) : s(src), icase(ic) {}

    int add(Ast a)
    {
        nodes.push_back(std::move(a));
        return (int)nodes.size() - 1;
    }
    int refuse(const char *msg)
    {
        if (why.empty()) why = msg;
        return -1;
    }
    int leaf(Ast::Kind k)
    {
        Ast a;
        a.kind = k;
        return add(a);
    }
    int set_node(CharSet cs, bool from_bracket)
    {
        if (icase)
        {
            CharSet c2 = cs;
            for (int c = 'A'; c <= 'Z'; c++)
                if (cs[c] || cs[c + 32]) c2[c] = c2[c + 32] = true;
            if (from_bracket && c2 != cs) widened = true; // glibc's -i bracket rules are not modelled: take the case closure
            cs = c2;
        }
        if (cs['\n']) return refuse("a character set of the pattern contains the newline");
        Ast a;
        a.kind = Ast::SET;
        a.set = cs;
        return add(a);
    }

    int parse_alt()
    {
        std::vector<int> br{parse_cat()};
        while (br.back() >= 0 && i < s.size() && s[i] == '|')
        {
            i++;
            br.push_back(parse_cat());
        }
        if (br.back() < 0) return -1;
        if (br.size() == 1) return br[0];
        Ast a;
        a.kind = Ast::ALT;
        a.kids = br;
        return add(a);
    }

    int parse_cat()
    {
        std::vector<int> items;
        while (i < s.size() && s[i] != '|' && s[i] != ')')
        {
            int r = parse_repeat();
            if (r < 0) return -1;
            items.push_back(r);
        }
        if (items.empty()) return leaf(Ast::EMPTY);
        if (items.size() == 1) return items[0];
        Ast a;
        a.kind = Ast::CAT;
        a.kids = items;
        return add(a);
    }

    bool number(int *v)
    {
        if (i >= s.size() || s[i] < '0' || s[i] > '9') return false;
        long x = 0;
        while (i < s.size() && s[i] >= '0' && s[i] <= '9')
        {
            x = x * 10 + (s[i++] - '0');
            if (x > 255) return false; // larger counts: refused (the expansion would exceed the automaton budget anyway)
        }
        *v = (int)x;
        return true;
    }

    int parse_repeat()
    {
        int atom = parse_atom();
        while (atom >= 0 && i < s.size())
        {
            int mn, mx;
            const char c = s[i];
            if (c == '*') mn = 0, mx = -1, i++;
            else if (c == '+') mn = 1, mx = -1, i++;
            else if (c == '?') mn = 0, mx = 1, i++;
            else if (c == '{')
            {
                i++;
                mn = 0;
                const bool has_min = number(&mn);
                if (i < s.size() && s[i] == '}')
                {
                    if (!has_min) return refuse("empty interval");
                    mx = mn;
                }
                else if (i < s.size() && s[i] == ',')
                {
                    i++;
                    mx = -1;
                    if (i < s.size() && s[i] != '}' && !number(&mx)) return refuse("interval bound");
                }
                else return refuse("interval");
                if (i >= s.size() || s[i] != '}') return refuse("interval");
                i++;
                if (mx >= 0 && mx < mn) return refuse("interval bounds");
            }
            else break;
            Ast a;
            a.kind = Ast::REP;
            a.kids = {atom};
            a.min = mn;
            a.max = mx;
            atom = add(a);
        }
        return atom;
    }

    int parse_atom()
    {
        const unsigned char c = (unsigned char)s[i];
        switch (c)
        {
        case '(':
        {
            i++;
            int r = parse_alt();
            if (r < 0) return -1;
            if (i >= s.size() || s[i] != ')') return refuse("unbalanced parenthesis");
            i++;
            return r;
        }
        case ')': return refuse("unmatched ')'");
        case '*': case '+': case '?': case '{': return refuse("repetition without an operand");
        case '^': i++; return leaf(Ast::BOL);
        case '$': i++; return leaf(Ast::EOL);
        case '.':
        {
            i++;
            CharSet cs;
            cs.set();
            cs['\n'] = false; // REG_NEWLINE
            cs[0] = false;    // RE_DOT_NOT_NULL (POSIX syntax)
            return set_node(cs, false);
        }
        case '[': i++; return parse_bracket();
        case '\\': i++; return parse_escape();
        default:
        {
            i++;
            if (c == '\n') return refuse("newline in the pattern");
            if (c >= 0x80) return refuse("non-ASCII byte in the pattern");
            CharSet cs;
            cs[c] = true;
            return set_node(cs, false);
        }
        }
    }

    int parse_escape()
    {
        if (i >= s.size()) return refuse("trailing backslash");
        const unsigned char c = (unsigned char)s[i++];
        CharSet cs;
        switch (c)
        {
        case 'b': case 'B': case '<': case '>':
            widened = true; // word assertions: matched by the empty string (a wider answer, see the file comment)
            return leaf(Ast::EMPTY);
        case 'w':
            for (int k = 0; k < 256; k++) cs[k] = is_word_c(k);
            return set_node(cs, false);
        case 'W': case 's': case 'S': case '`': case '\'':
            // \W and \s match '\n' (even under REG_NEWLINE); \S is left out with them; \` \' are buffer anchors
            return refuse("unsupported escape");
        default:
            if (c >= '1' && c <= '9') return refuse("back-reference");
            if ((c >= 'a' && c <= 'z') || (c >= 'A' && c <= 'Z') || (c >= '0' && c <= '9') || c >= 0x80 || c == '\n')
                return refuse("unknown escape");
            cs[c] = true; // an escaped punctuation character stands for itself
            return set_node(cs, false);
        }
    }

    bool char_class(const std::string &name, CharSet *cs)
    {
        for (int k = 0; k < 128; k++)
        {
            bool in;
            if (name == "alpha") in = is_alpha_c(k);
            else if (name == "digit") in = k >= '0' && k <= '9';
            else if (name == "alnum") in = is_alpha_c(k) || (k >= '0' && k <= '9');
            else if (name == "upper") in = k >= 'A' && k <= 'Z';
            else if (name == "lower") in = k >= 'a' && k <= 'z';
            else if (name == "blank") in = k == ' ' || k == '\t';
            else if (name == "punct") in = k > 32 && k < 127 && !is_alpha_c(k) && !(k >= '0' && k <= '9');
            else if (name == "print") in = k >= 32 && k < 127;
            else if (name == "graph") in = k > 32 && k < 127;
            else if (name == "xdigit") in = (k >= '0' && k <= '9') || (k >= 'a' && k <= 'f') || (k >= 'A' && k <= 'F');
            else return false; // space / cntrl hold '\n'; anything else is unknown
            if (in) (*cs)[k] = true;
        }
        return true;
    }

    // glibc's set of the bracket expression src under -i.  POSIX leaves case-insensitive ranges to the implementation,
    // and glibc's answer is not the case closure of the range ([A-z] holds no byte of [\]^_`, [a-|] holds all six), so
    // glibc is asked itself: the bracket alone, compiled as krep compiles -i regexes, against every byte but the newline.
    // false when glibc refuses the bracket.
    static bool icase_bracket(const std::string &src, CharSet *cs)
    {
        regex_t rx;
        if (regcomp(&rx, src.c_str(), REG_EXTENDED | REG_NEWLINE | REG_ICASE) != 0) return false;
        cs->reset();
        for (int b = 0; b < 256; b++)
        {
            if (b == '\n') continue;
            const char c = (char)b;
            regmatch_t m;
            m.rm_so = 0;
            m.rm_eo = 1; // REG_STARTEND: the one byte, NUL included
            if (regexec(&rx, &c, 1, &m, REG_STARTEND) == 0) (*cs)[b] = true;
        }
        regfree(&rx);
        return true;
    }

    int parse_bracket()
    {
        const size_t open = i - 1; // the '['
        CharSet cs;
        bool neg = false;
        if (i < s.size() && s[i] == '^') neg = true, i++;
        bool first = true;
        for (;;)
        {
            if (i >= s.size()) return refuse("unterminated bracket expression");
            unsigned char c = (unsigned char)s[i];
            if (c == ']' && !first)
            {
                i++;
                break;
            }
            first = false;
            if (c == '[' && i + 1 < s.size() && (s[i + 1] == '.' || s[i + 1] == '=')) return refuse("collating element");
            if (c == '[' && i + 1 < s.size() && s[i + 1] == ':')
            {
                const size_t e = s.find(":]", i + 2);
                if (e == std::string::npos || !char_class(s.substr(i + 2, e - i - 2), &cs)) return refuse("character class");
                i = e + 2;
                if (i < s.size() && s[i] == '-' && i + 1 < s.size() && s[i + 1] != ']') return refuse("range from a class");
                continue;
            }
            if (c >= 0x80) return refuse("non-ASCII byte in the pattern");
            i++;
            if (i + 1 < s.size() && s[i] == '-' && s[i + 1] != ']')
            {
                const unsigned char d = (unsigned char)s[i + 1];
                if (d == '[' || d >= 0x80 || d < c) return refuse("range");
                i += 2;
                for (int k = c; k <= d; k++) cs[k] = true;
            }
            else cs[c] = true;
        }
        if (neg)
        {
            cs.flip();
            cs['\n'] = false; // REG_NEWLINE: a non-matching list never matches the newline
        }
        // under -i, set_node decides refusal and widening from the case closure of the parsed set, as for every other
        // set; the bytes the automaton reads are glibc's
        const int n = set_node(cs, true);
        if (n >= 0 && icase && !icase_bracket(s.substr(open, i - open), &nodes[n].set))
            return refuse("a bracket expression glibc refuses under -i");
        return n;
    }
};

// ---- Thompson NFA ------------------------------------------------------------------------------------------------
struct NState
{
    enum Kind { CHAR, SPLIT, BOL, EOL, MATCH } kind;
    int set = -1;      // CHAR: index into Nfa::sets
    int out = -1, out1 = -1;
};

struct Nfa
{
    std::vector<NState> st;
    std::vector<CharSet> sets;
    bool too_big = false;
    bool widened = false;
    static constexpr size_t MAX_STATES = 8192;

    int add(NState::Kind k)
    {
        if (st.size() >= MAX_STATES) too_big = true;
        st.push_back(NState{k});
        return (int)st.size() - 1;
    }
    // Fragment: entry state and the list of dangling exits (state index, which out)
    struct Frag
    {
        int in;
        std::vector<std::pair<int, int>> outs;
    };
    void patch(const Frag &f, int to)
    {
        for (auto &o : f.outs) (o.second ? st[o.first].out1 : st[o.first].out) = to;
    }
    // in_rep: inside a repeated group, where glibc's anchors do not behave as anchors (it matches "(^a){2}" on "aa"):
    // ^ and $ there are built as empty (a wider answer)
    Frag build(const std::vector<Ast> &A, int n, bool in_rep = false)
    {
        if (too_big) return Frag{add(NState::SPLIT), {}};
        const Ast &a = A[n];
        switch (a.kind)
        {
        case Ast::SET:
        {
            int s = add(NState::CHAR);
            st[s].set = (int)sets.size();
            sets.push_back(a.set);
            return Frag{s, {{s, 0}}};
        }
        case Ast::BOL: case Ast::EOL: case Ast::EMPTY:
        {
            if (in_rep && a.kind != Ast::EMPTY) widened = true;
            const NState::Kind k = in_rep ? NState::SPLIT : a.kind == Ast::BOL ? NState::BOL : a.kind == Ast::EOL ? NState::EOL : NState::SPLIT;
            int s = add(k);
            return Frag{s, {{s, 0}}}; // an EMPTY split has out1 = -1: a plain epsilon edge
        }
        case Ast::CAT:
        {
            Frag f = build(A, a.kids[0], in_rep);
            for (size_t k = 1; k < a.kids.size(); k++)
            {
                Frag g = build(A, a.kids[k], in_rep);
                patch(f, g.in);
                f.outs = g.outs;
            }
            return f;
        }
        case Ast::ALT:
        {
            Frag f = build(A, a.kids[0], in_rep);
            for (size_t k = 1; k < a.kids.size(); k++)
            {
                Frag g = build(A, a.kids[k], in_rep);
                int s = add(NState::SPLIT);
                st[s].out = f.in;
                st[s].out1 = g.in;
                f.in = s;
                f.outs.insert(f.outs.end(), g.outs.begin(), g.outs.end());
            }
            return f;
        }
        case Ast::REP:
        default:
        {
            // x{m,n} = x^m (x?)^(n-m);  x{m,} = x^m x*;  each copy is a fresh fragment
            int entry = add(NState::SPLIT); // epsilon entry (keeps zero-repetition cases uniform)
            Frag f{entry, {{entry, 0}}};
            const bool rep = in_rep || a.max != 1 || a.min > 1;
            for (int k = 0; k < a.min; k++)
            {
                Frag g = build(A, a.kids[0], rep);
                patch(f, g.in);
                f.outs = g.outs;
            }
            if (a.max < 0)
            {
                Frag g = build(A, a.kids[0], rep);
                int s = add(NState::SPLIT);
                st[s].out = g.in;
                patch(g, s);
                patch(f, s);
                f.outs = {{s, 1}};
            }
            else
            {
                std::vector<std::pair<int, int>> exits;
                for (int k = a.min; k < a.max; k++)
                {
                    Frag g = build(A, a.kids[0], rep);
                    int s = add(NState::SPLIT);
                    st[s].out = g.in;
                    patch(f, s);
                    exits.push_back({s, 1});
                    f.outs = g.outs;
                }
                f.outs.insert(f.outs.end(), exits.begin(), exits.end());
            }
            return f;
        }
        }
    }
};

// epsilon closure of `seed` (sorted, unique result).  BOL edges are followed only at the start of the line, EOL edges
// only when `at_eol`.  *match = MATCH was reached.
void closure(const Nfa &N, std::vector<int> seed, bool at_bol, bool at_eol, std::vector<int> *out, bool *match)
{
    std::vector<char> seen(N.st.size(), 0);
    out->clear();
    *match = false;
    while (!seed.empty())
    {
        int s = seed.back();
        seed.pop_back();
        if (s < 0 || seen[s]) continue;
        seen[s] = 1;
        const NState &x = N.st[s];
        switch (x.kind)
        {
        case NState::CHAR: out->push_back(s); break;
        case NState::MATCH: *match = true; break;
        case NState::SPLIT: seed.push_back(x.out); seed.push_back(x.out1); break;
        case NState::BOL: if (at_bol) seed.push_back(x.out); break;
        case NState::EOL:
            if (at_eol) seed.push_back(x.out);
            else out->push_back(s); // kept: the line may end right here
            break;
        }
    }
    std::sort(out->begin(), out->end());
}

// The anchored match automaton of an exact plan (DESIGN §12.2): the subset construction of R itself — no restart
// closure, so a walk from a start position reads the matches that begin there — over the byte classes of the line
// table.  Two start states: at the line's first byte (BOL edges followed) and anywhere else (not followed).  State 0 is
// DEAD.  Returns false when the table would not fit `budget_entries`: the plan then keeps its offsets on regexec.
bool build_match_automaton(const Nfa &N, int start, const uint8_t *cls, int nc, const std::vector<int> &rep,
                           size_t budget_entries, RegexDfa *D)
{
    const int nl = cls['\n'];
    std::vector<std::vector<int>> sets(1); // [0] = DEAD (the empty set)
    std::vector<char> is_bol(1, 0);
    std::map<std::pair<std::vector<int>, int>, int> index; // (set, bol | matched << 1)
    index.emplace(std::make_pair(std::vector<int>(), 0), 0);
    std::vector<uint16_t> acc(1, 0);
    auto intern = [&](std::vector<int> set, bool bol, bool matched) -> int {
        auto key = std::make_pair(set, (bol ? 1 : 0) | (matched ? 2 : 0));
        auto it = index.find(key);
        if (it != index.end()) return it->second;
        sets.push_back(std::move(set));
        is_bol.push_back(bol ? 1 : 0);
        acc.push_back(matched ? RX_ACC : 0);
        index.emplace(key, (int)sets.size() - 1);
        return (int)sets.size() - 1;
    };
    std::vector<int> s0;
    bool m0 = false;
    closure(N, {start}, true, false, &s0, &m0);
    const int bol_state = intern(s0, true, m0);
    closure(N, {start}, false, false, &s0, &m0);
    const int mid_state = intern(s0, false, m0);
    std::vector<std::vector<int>> next(1, std::vector<int>(nc, 0));
    for (size_t s = 1; s < sets.size(); s++)
    {
        if (sets.size() * (size_t)nc > budget_entries) return false;
        // accepts if the line ends here: a match that ends here anyway, or one through EOL edges (the set keeps the EOL
        // states; BOL edges are followed at the line start)
        if (acc[s] & RX_ACC) acc[s] |= RX_ACC_EOL;
        else
        {
            std::vector<int> seed = sets[s], tmp;
            if (is_bol[s]) seed.push_back(start);
            bool a = false;
            closure(N, seed, is_bol[s], true, &tmp, &a);
            if (a) acc[s] |= RX_ACC_EOL;
        }
        std::vector<int> row(nc, 0);
        for (int c = 0; c < nc; c++)
        {
            if (c == nl) continue; // holds the accept bits
            const int b = rep[c];
            std::vector<int> moved;
            for (int x : sets[s])
                if (N.st[x].kind == NState::CHAR && N.sets[N.st[x].set][b]) moved.push_back(N.st[x].out);
            if (moved.empty()) continue;
            std::vector<int> cl;
            bool mt = false;
            closure(N, moved, false, false, &cl, &mt);
            row[c] = intern(cl, false, mt);
        }
        next.push_back(row);
    }
    const size_t S = sets.size();
    if (S * (size_t)nc > budget_entries) return false;
    D->match.assign(S * nc, 0);
    for (size_t s = 0; s < S; s++)
        for (int c = 0; c < nc; c++)
            D->match[s * nc + c] = c == nl ? acc[s] : (uint16_t)(next[s][c] * nc);
    D->match_bol = (uint32_t)(bol_state * nc);
    D->match_mid = (uint32_t)(mid_state * nc);
    return true;
}

} // namespace

// The regular expression krep hands to regcomp (krep.c:2081-2145 and 2539-2600): patterns are read as C strings.
bool regex_source(const search_params_t *P, std::string *out)
{
    if (!P || P->num_patterns == 0 || !P->patterns) return false;
    std::string r;
    if (P->num_patterns > 1)
    {
        for (size_t k = 0; k < P->num_patterns; k++)
        {
            const char *p = P->patterns[k] ? P->patterns[k] : "";
            r += P->whole_word ? std::string("(\\b") + p + "\\b)" : std::string("(") + p + ")";
            if (k + 1 < P->num_patterns) r += "|";
        }
    }
    else
    {
        const char *p = P->patterns[0] ? P->patterns[0] : "";
        r = P->whole_word ? std::string("\\b") + p + "\\b" : std::string(p);
    }
    *out = r;
    return true;
}

namespace {

// The automata of the regex rooted at node `root` of a parse: its line automaton and, when its per-line answer is exact,
// its anchored match automaton.  Every refusal here is one of size (states, table bytes, NFA states, byte classes).
// parse_widened: the parse widened a set or an assertion.  max_states: REGEX_MAX_STATES, or a smaller test cap.
// smem_bytes: the shared memory its line table, class map and match table may take together (a split plan checks the
// sum over its automata afterwards); 0 builds the line automaton only.
int compile_automaton(const std::vector<Ast> &nodes, int root, bool parse_widened, uint32_t max_states, size_t smem_bytes,
                      RegexDfa *D, std::string *why)
{
    Nfa N;
    Nfa::Frag f = N.build(nodes, root);
    int m = N.add(NState::MATCH);
    N.patch(f, m);
    if (N.too_big)
    {
        *why = "the automaton is too large";
        return -1;
    }
    const int start = f.in;

    // byte classes: bytes that every character set of the pattern treats alike; '\n' is a class of its own
    std::map<std::vector<bool>, int> sig_class;
    uint8_t cls[256];
    for (int b = 0; b < 256; b++)
    {
        std::vector<bool> sig(N.sets.size() + 1);
        for (size_t k = 0; k < N.sets.size(); k++) sig[k] = N.sets[k][b];
        sig[N.sets.size()] = b == '\n';
        auto it = sig_class.find(sig);
        if (it == sig_class.end()) it = sig_class.emplace(sig, (int)sig_class.size()).first;
        cls[b] = (uint8_t)it->second;
    }
    const int nc = (int)sig_class.size();
    if (nc > 255)
    {
        *why = "too many byte classes";
        return -1;
    }
    std::vector<int> rep(nc, 0); // one byte of each class
    for (int b = 255; b >= 0; b--) rep[cls[b]] = b;

    // subset construction of the unanchored line automaton [^\n]*R.  DFA state 0 = MATCHED (the line is flagged), 1 =
    // DEAD (no match can start or end anywhere in the rest of the line); the line-start state comes next.
    struct DState
    {
        std::vector<int> set;
        bool bol;
    };
    std::vector<DState> states(2);
    std::map<std::pair<std::vector<int>, bool>, int> index;
    std::vector<std::vector<int>> next; // next[s][c]
    std::vector<char> eol_acc;          // accepts when the line ends here
    std::vector<int> restart;
    bool restart_match = false;
    closure(N, {start}, false, false, &restart, &restart_match);

    auto intern = [&](std::vector<int> set, bool bol, bool matched) -> int {
        if (matched) return 0;
        auto key = std::make_pair(set, bol);
        auto it = index.find(key);
        if (it != index.end()) return it->second;
        states.push_back(DState{std::move(set), bol});
        index.emplace(key, (int)states.size() - 1);
        return (int)states.size() - 1;
    };
    std::vector<int> s0;
    bool m0 = false;
    closure(N, {start}, true, false, &s0, &m0);
    const int start_state = intern(s0, true, m0);
    const size_t budget_entries = REGEX_TABLE_BYTES / sizeof(uint16_t);
    next.assign(2, std::vector<int>(nc, 0));
    eol_acc.assign(2, 0);
    eol_acc[0] = 1;
    for (int c = 0; c < nc; c++) next[1][c] = 1;
    for (size_t s = 2; s < states.size(); s++)
    {
        if (states.size() * (size_t)nc > budget_entries || states.size() > max_states)
        {
            *why = "the automaton has too many states";
            return -1;
        }
        const std::vector<int> set = states[s].set;
        const bool bol = states[s].bol;
        // end of line here?
        {
            std::vector<int> seed = set, tmp;
            if (bol) seed.push_back(start);
            bool acc = false;
            closure(N, seed, bol, true, &tmp, &acc);
            eol_acc.push_back(acc ? 1 : 0);
        }
        std::vector<int> row(nc, 1);
        for (int c = 0; c < nc; c++)
        {
            if (c == cls['\n']) continue; // the kernel reads the '\n' column as "accepts at end of line"
            const int b = rep[c];
            std::vector<int> moved = restart;
            for (int x : set)
                if (N.st[x].kind == NState::CHAR && N.sets[N.st[x].set][b]) moved.push_back(N.st[x].out);
            std::vector<int> cl;
            bool mt = false;
            closure(N, moved, false, false, &cl, &mt);
            row[c] = intern(cl, false, mt);
        }
        next.push_back(row);
    }
    const int S = (int)states.size();
    // states from which no match is reachable within the line behave like DEAD
    std::vector<char> live(S, 0);
    live[0] = 1;
    for (bool changed = true; changed;)
    {
        changed = false;
        for (int s = 2; s < S; s++)
        {
            if (live[s]) continue;
            bool l = eol_acc[s];
            for (int c = 0; c < nc && !l; c++) l = c != cls['\n'] && live[next[s][c]];
            if (l) live[s] = 1, changed = true;
        }
    }
    D->nclasses = (uint32_t)nc;
    D->nl_class = cls['\n'];
    memcpy(D->cls, cls, 256);
    D->nstates = (uint32_t)S;
    D->start = (uint32_t)((live[start_state] ? start_state : 1) * nc);
    D->trans.assign((size_t)S * nc, 0);
    for (int s = 0; s < S; s++)
        for (int c = 0; c < nc; c++)
        {
            int t;
            if (s == 0) t = 0;
            else if (c == cls['\n']) t = eol_acc[s] ? 0 : 1;
            else t = live[next[s][c]] ? next[s][c] : 1;
            D->trans[(size_t)s * nc + c] = (uint16_t)(t * nc); // entries are row offsets: next = trans[row + class]
        }
    D->widened = parse_widened || N.widened;
    D->count_exact = !D->widened;
    // offsets on the device: the plans whose per-line answer is exact, when the match automaton fits the shared memory
    // left next to the line table and the class map
    D->offsets_exact = false;
    if (D->count_exact && smem_bytes)
    {
        const size_t used = (size_t)regex_tab_words((uint32_t)D->trans.size()) * 2 + 256;
        // entries are 16-bit row offsets: a table of more than 65536 entries could not address its last rows
        const size_t budget = std::min<size_t>(used < smem_bytes ? (smem_bytes - used) / 2 : 0, 65536);
        D->offsets_exact = build_match_automaton(N, start, cls, nc, rep, budget & ~(size_t)7, D);
        if (!D->offsets_exact) D->match.clear();
    }
    return 0;
}

// A split plan (DESIGN §12.7) of the top-level alternation `root`: its branches, in order, packed greedily into groups
// of as many consecutive branches as one automaton holds (found by doubling the group, then bisecting), at most
// REGEX_MAX_GROUPS of them, all in one image of REGEX_SET_SMEM_BYTES.  The packing compiles line automata only and
// gives up as soon as the groups placed so far exceed the image or the group count; the match automata are built once,
// for the final groups.  A group's match automaton may use what the image leaves; the sum over the groups decides
// whether offsets stay on the device.
int compile_split(std::vector<Ast> nodes, int root, bool parse_widened, uint32_t max_states, RegexDfa *D, std::string *why)
{
    const std::vector<int> br = nodes[root].kids;
    auto compile_group = [&](size_t i, size_t k, RegexDfa *G, size_t smem_bytes) { // branches [i, i + k)
        int r = br[i];
        if (k > 1)
        {
            Ast a;
            a.kind = Ast::ALT;
            a.kids.assign(br.begin() + i, br.begin() + i + k);
            nodes.push_back(a);
            r = (int)nodes.size() - 1;
        }
        std::string w;
        const bool ok = compile_automaton(nodes, r, parse_widened, max_states, smem_bytes, G, &w) == 0;
        if (k > 1) nodes.pop_back();
        return ok;
    };
    std::vector<RegexDfa> groups;
    std::vector<std::pair<size_t, size_t>> spans; // the branches [first, first + count) of each group
    size_t line_bytes = 0;
    for (size_t i = 0; i < br.size();)
    {
        const size_t left = br.size() - i;
        if (groups.size() == REGEX_MAX_GROUPS)
        {
            *why = "the alternation needs more automata than a split plan holds";
            return -1;
        }
        RegexDfa best;
        if (!compile_group(i, 1, &best, 0))
        {
            *why = "a branch of the alternation is too large for one automaton";
            return -1;
        }
        size_t ok = 1, bad = i == 0 ? left : left + 1; // the whole alternation is known not to fit
        for (size_t k = 2; k < bad; k *= 2)
        {
            RegexDfa g;
            const size_t kk = std::min(k, left);
            if (!compile_group(i, kk, &g, 0))
            {
                bad = kk;
                break;
            }
            ok = kk;
            best = std::move(g);
            if (kk == left) break;
        }
        while (ok < left && bad - ok > 1)
        {
            RegexDfa g;
            const size_t mid = ok + (bad - ok) / 2;
            if (compile_group(i, mid, &g, 0)) ok = mid, best = std::move(g);
            else bad = mid;
        }
        line_bytes += (size_t)regex_tab_words((uint32_t)best.trans.size()) * 2 + 256;
        if (line_bytes > REGEX_SET_SMEM_BYTES)
        {
            *why = "the automata of the alternation exceed the shared memory of one scan";
            return -1;
        }
        groups.push_back(std::move(best));
        spans.push_back({i, ok});
        i += ok;
    }
    bool widened = false;
    for (const RegexDfa &g : groups) widened |= g.widened;
    size_t match_bytes = 0;
    bool matches = !widened;
    for (size_t g = 0; g < groups.size() && matches; g++)
    {
        // the same line automaton again, now with its match automaton
        matches = compile_group(spans[g].first, spans[g].second, &groups[g], REGEX_SET_SMEM_BYTES) && groups[g].offsets_exact;
        match_bytes += (size_t)regex_tab_words((uint32_t)groups[g].match.size()) * 2;
    }
    D->widened = widened;
    D->count_exact = !widened;
    D->offsets_exact = D->count_exact && matches && line_bytes + match_bytes <= REGEX_SET_SMEM_BYTES;
    if (!D->offsets_exact)
        for (RegexDfa &g : groups) g.offsets_exact = false, g.match.clear();
    D->groups = std::move(groups);
    return 0;
}

} // namespace

int regex_compile(const std::string &re, bool icase, RegexDfa *D, std::string *why, uint32_t max_states)
{
    if (MB_CUR_MAX != 1)
    {
        // krep never calls setlocale: its regexes are C-locale regexes.  A host running in a multibyte locale compiled
        // a regex whose '.' and brackets match characters of several bytes, which a byte automaton does not model.
        *why = "the process runs in a multibyte locale";
        return -1;
    }
    Parser ps(re, icase);
    int root = ps.parse_alt();
    if (root >= 0 && ps.i != re.size()) root = ps.refuse("unmatched ')'");
    if (root < 0)
    {
        *why = ps.why;
        return -1;
    }
    // a regex one automaton holds is compiled as one; an alternation too large for one is split at its top level
    if (compile_automaton(ps.nodes, root, ps.widened, max_states, REGEX_SMEM_BYTES, D, why) == 0) return 0;
    if (ps.nodes[root].kind != Ast::ALT) return -1;
    std::string whole = *why;
    if (compile_split(std::move(ps.nodes), root, ps.widened, max_states, D, why) == 0) return 0;
    *why = whole + "; " + *why;
    return -1;
}

void regex_layout(const RegexDfa &D, RegexGroup *grp, uint32_t *ngroups, uint32_t *line_words, uint32_t *image_words)
{
    std::vector<const RegexDfa *> au;
    if (D.groups.empty()) au.push_back(&D);
    for (const RegexDfa &g : D.groups) au.push_back(&g);
    uint32_t w = 0;
    for (size_t g = 0; g < au.size(); g++)
    {
        grp[g].trans = w;
        w += regex_tab_words((uint32_t)au[g]->trans.size());
        grp[g].cls = w;
        w += 128;
        grp[g].nclasses = au[g]->nclasses;
        grp[g].nl_class = au[g]->nl_class;
        grp[g].start = au[g]->start;
        grp[g].match_bol = au[g]->match_bol;
        grp[g].match_mid = au[g]->match_mid;
    }
    *line_words = w;
    for (size_t g = 0; g < au.size(); g++)
    {
        grp[g].match = w;
        w += regex_tab_words((uint32_t)au[g]->match.size());
    }
    *image_words = w;
    *ngroups = (uint32_t)au.size();
    for (size_t g = au.size(); g < REGEX_MAX_GROUPS; g++)
    {
        // spare slots of the kernel's automata: the first group's, started DEAD (in both tables)
        grp[g] = grp[0];
        grp[g].start = grp[0].nclasses;
        grp[g].match_bol = grp[g].match_mid = 0;
    }
}

std::vector<uint16_t> regex_image(const RegexDfa &D)
{
    RegexGroup grp[REGEX_MAX_GROUPS];
    uint32_t ng, lw, iw;
    regex_layout(D, grp, &ng, &lw, &iw);
    std::vector<uint16_t> img(iw, 0);
    for (uint32_t g = 0; g < ng; g++)
    {
        const RegexDfa &A = D.groups.empty() ? D : D.groups[g];
        std::copy(A.trans.begin(), A.trans.end(), img.begin() + grp[g].trans);
        memcpy(img.data() + grp[g].cls, A.cls, 256);
        std::copy(A.match.begin(), A.match.end(), img.begin() + grp[g].match);
    }
    return img;
}

namespace {

// The line walk of a plan on the host, over its one automaton or the automata of a split plan: the line is MATCHED as
// soon as one automaton is, DEAD once all are.
struct LineWalk
{
    std::vector<const RegexDfa *> au;
    std::vector<uint32_t> r;
    enum { MATCHED, DEAD, LIVE } state = LIVE;

    explicit LineWalk(const RegexDfa &D)
    {
        if (D.groups.empty()) au.push_back(&D);
        for (const RegexDfa &g : D.groups) au.push_back(&g);
        r.resize(au.size());
    }
    void settle()
    {
        state = DEAD;
        for (size_t g = 0; g < au.size(); g++)
        {
            if (r[g] == 0)
            {
                state = MATCHED;
                return;
            }
            if (r[g] > au[g]->nclasses) state = LIVE;
        }
    }
    void begin()
    {
        for (size_t g = 0; g < au.size(); g++) r[g] = au[g]->start;
        settle();
    }
    void step(uint8_t b)
    {
        for (size_t g = 0; g < au.size(); g++) r[g] = au[g]->trans[r[g] + au[g]->cls[b]];
        settle();
    }
    void end_of_line() // the '\n' column of every live automaton
    {
        for (size_t g = 0; g < au.size(); g++)
            if (r[g] > au[g]->nclasses) r[g] = au[g]->trans[r[g] + au[g]->nl_class];
        settle();
    }
};

} // namespace

// The line filter run on the host — what k_regex_lines computes, without the kernel's long-line bound.
void regex_lines_host(const RegexDfa &D, const char *t, size_t n, std::vector<uint64_t> *out)
{
    out->clear();
    LineWalk W(D);
    size_t p = 0;
    while (p < n)
    {
        W.begin();
        size_t q = p;
        for (; q < n && t[q] != '\n' && W.state == LineWalk::LIVE; q++) W.step((uint8_t)t[q]);
        if (W.state == LineWalk::LIVE) W.end_of_line(); // end of line (or of the text)
        if (W.state == LineWalk::MATCHED) out->push_back(p);
        const void *nl = q < n ? memchr(t + q, '\n', n - q) : nullptr;
        if (!nl) break;
        p = (size_t)((const char *)nl - t) + 1;
    }
}

// The count mode of k_regex_lines (scan_regex.cu), one line at a time.  The kernel's walk ends REGEX_HALO bytes past its
// thread's segment; here every line may be read `reach` bytes from its start (UINT64_MAX: to the end of the text), so a
// small reach drives the uncertain-line path without a GPU.
uint64_t regex_count_lines_host(const RegexDfa &D, const char *t, size_t n, uint64_t reach, std::vector<uint64_t> *uncertain)
{
    uncertain->clear();
    LineWalk W(D);
    uint64_t counted = 0;
    size_t p = 0;
    while (p < n)
    {
        const size_t limit = reach < n - p ? p + (size_t)reach : n;
        W.begin();
        size_t q = p;
        for (; q < limit && t[q] != '\n' && W.state == LineWalk::LIVE; q++) W.step((uint8_t)t[q]);
        if (W.state == LineWalk::LIVE && q < limit) W.end_of_line(); // the walk stopped at the line's '\n'
        if (W.state != LineWalk::LIVE)
            while (q < limit && t[q] != '\n') q++;
        if (q >= limit || q + 1 == n) uncertain->push_back(p); // '\n' out of reach, or the text's last byte
        else if (W.state == LineWalk::MATCHED) counted++;
        const void *nl = q < n ? memchr(t + q, '\n', n - q) : nullptr;
        if (!nl) break;
        p = (size_t)((const char *)nl - t) + 1;
    }
    return counted;
}

// The match mode of k_regex_lines (scan_regex.cu): the line walk of the count mode, then for a line decided MATCHED the
// reference's loop restated inside the line [p, q] (q = its '\n'): from cur, the leftmost start s with a match and its
// longest end e, emitted; cur = e, or s + 1 after an empty match; until cur passes q.  '^' holds only at s == p, '$'
// only at q.  A split plan tries every automaton at s: the match starts at the first s where one accepts and ends at the
// longest of their ends, with G times the budget of one automaton.  A line whose enumeration runs over its step budget,
// or finds a match of REGEX_LONG_MAX_MATCH bytes or more (only lines past the kernel's reach have one; the long-line
// pass does the same), leaves an uncertain key behind the match keys it already emitted (the host drops those).
void regex_matches_host(const RegexDfa &D, const char *t, size_t n, uint64_t reach, std::vector<uint64_t> *keys)
{
    keys->clear();
    LineWalk W(D);
    size_t p = 0;
    while (p < n)
    {
        const size_t limit = reach < n - p ? p + (size_t)reach : n;
        W.begin();
        size_t q = p;
        for (; q < limit && t[q] != '\n' && W.state == LineWalk::LIVE; q++) W.step((uint8_t)t[q]);
        if (W.state == LineWalk::LIVE && q < limit) W.end_of_line();
        if (W.state != LineWalk::LIVE)
            while (q < limit && t[q] != '\n') q++;
        if (q >= limit || q + 1 == n) keys->push_back((uint64_t)p << REGEX_MATCH_SHIFT);
        else if (W.state == LineWalk::MATCHED)
        {
            const uint64_t budget = W.au.size() * ((uint64_t)REGEX_MATCH_STEPS_PER_BYTE * (q - p) + REGEX_MATCH_STEPS_BASE);
            uint64_t steps = 0;
            size_t cur = p;
            bool flag = false;
            while (cur <= q && steps <= budget)
            {
                size_t s = cur, e = 0;
                bool found = false;
                for (; s <= q && steps <= budget; s++)
                {
                    for (const RegexDfa *A : W.au)
                    {
                        const uint16_t *M = A->match.data();
                        const uint32_t nl = A->nl_class;
                        uint32_t r = s == p ? A->match_bol : A->match_mid;
                        steps++;
                        if (M[r + nl] & (s == q ? RX_ACC_EOL : RX_ACC)) found = true, e = std::max(e, s);
                        for (size_t x = s; x < q && r != 0;)
                        {
                            r = M[r + A->cls[(uint8_t)t[x++]]];
                            steps++;
                            if (M[r + nl] & (x == q ? RX_ACC_EOL : RX_ACC)) found = true, e = std::max(e, x);
                        }
                    }
                    if (found) break;
                }
                if (!found) break;
                if (e - s >= REGEX_LONG_MAX_MATCH)
                {
                    flag = true; // the match does not fit the key's length field: the line goes to regexec whole
                    break;
                }
                keys->push_back(((uint64_t)s << REGEX_MATCH_SHIFT) | ((uint64_t)(e - s) << LIT_TAG_BITS) | 1);
                cur = e == s ? s + 1 : e;
            }
            if (flag || steps > budget) keys->push_back((uint64_t)p << REGEX_MATCH_SHIFT);
        }
        const void *nlp = q < n ? memchr(t + q, '\n', n - q) : nullptr;
        if (!nlp) break;
        p = (size_t)((const char *)nlp - t) + 1;
    }
    std::sort(keys->begin(), keys->end());
}

} // namespace kb
