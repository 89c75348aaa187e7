// Native front door: the compiled-program file (`out`), the witness file and the statement schedule.
//
// Replaces, on the host side of the C ABI, what `zokrates generate-proof` / `compute-witness` do before and after the
// arithmetic (all paths under /root/reference):
//   * `ProgEnum::deserialize` + `ProgHeader::read`      zokrates_ast/src/ir/serialize.rs:124-189,295-391   (header, four
//     sections, serde_cbor 0.11 statement stream: structs as text-keyed maps, externally tagged enums)
//   * `Computation::generate_constraints`                zokrates_ark/src/lib.rs:41-130   (IR -> R1CS in ark variable order:
//     index 0 = one, public arguments, then `~out_k` on first appearance are instance variables; private arguments, then
//     every other variable on first appearance scanning quad.left, quad.right, lin are witness variables; directives and
//     logs are skipped, :116)
//   * `Interpreter::execute_with_log_stream`             zokrates_interpreter/src/lib.rs:61-138   (statement order, the
//     assign-or-check rule for constraints, directives call a solver) — turned into a LEVEL schedule: the statements of
//     one dependency depth are independent and run as one kernel launch each (rows: ntt.cuh::witness_level_body,
//     directives: solver_body below)
//   * `Witness::read` / `Witness::write`                  zokrates_ast/src/ir/witness.rs:44-71   (usize LE count, then
//     (isize LE id, 32-byte canonical LE value) in BTreeMap order = ascending signed id)
// Pure host C++ (no CUDA): the same code runs in the CPU test build.
#pragma once
#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>
#include "rt.cuh"

namespace zkb {

enum SolverKind : uint32_t {   // zokrates_ast/src/common/solvers.rs:11-27
  SOLVER_CONDITION_EQ = 0, SOLVER_BITS = 1, SOLVER_DIV = 2, SOLVER_XOR = 3, SOLVER_OR = 4, SOLVER_SHA_AXXA = 5,
  SOLVER_SHA_CH = 6, SOLVER_EUCLIDEAN_DIV = 7, SOLVER_UNSUPPORTED = 255   // Zir / Sha256Round / SnarkVerifyBls12377: front-end gadgets
};
static constexpr uint32_t PROG_DIRECTIVE = 0x80000000u;   // statement list: constraint index, or this bit | directive index

// ---- CBOR (RFC 8949), the subset serde_cbor emits, read as a stream ---------------------------------------------------
struct Cbor {
  const uint8_t* d;
  size_t p, end;
  Cbor(const uint8_t* data, size_t pos, size_t e) : d(data), p(pos), end(e) {}
  [[noreturn]] static void bad(const char* what) { throw Error(ZKB_E_FORMAT, std::string("program file: ") + what); }
  uint8_t byte() { if (p >= end) bad("CBOR item runs past the end of its section"); return d[p++]; }
  const uint8_t* take(size_t n) { if (n > end - p) bad("CBOR item runs past the end of its section"); const uint8_t* q = d + p; p += n; return q; }
  // head of the next item: major type, argument; `indef` for indefinite lengths (argument meaningless then)
  void head(uint32_t& major, uint64_t& arg, bool& indef) {
    const uint8_t ib = byte();
    major = ib >> 5;
    const uint32_t info = ib & 31;
    indef = false;
    if (info < 24) { arg = info; return; }
    if (info == 24) { arg = byte(); return; }
    if (info == 25) { const uint8_t* q = take(2); arg = ((uint64_t)q[0] << 8) | q[1]; return; }
    if (info == 26) { const uint8_t* q = take(4); arg = 0; for (int i = 0; i < 4; i++) arg = (arg << 8) | q[i]; return; }
    if (info == 27) { const uint8_t* q = take(8); arg = 0; for (int i = 0; i < 8; i++) arg = (arg << 8) | q[i]; return; }
    if (info == 31) { indef = true; arg = 0; return; }
    bad("reserved CBOR additional information");
  }
  bool at_break() { return p < end && d[p] == 0xff; }
  void skip_tags() { while (p < end && (d[p] >> 5) == 6) { uint32_t m; uint64_t a; bool i; head(m, a, i); } }
  uint32_t depth = 0;
  void skip() {   // one complete item (nesting bounded: a hostile file must not overflow the stack)
    struct Guard { uint32_t& d; explicit Guard(uint32_t& x) : d(x) { if (++d > 128) bad("CBOR nesting too deep"); } ~Guard() { --d; } } g(depth);
    uint32_t major; uint64_t arg; bool indef;
    head(major, arg, indef);
    switch (major) {
      case 0: case 1: return;
      case 2: case 3:
        if (indef) { while (!at_break()) skip(); p++; } else take(arg);
        return;
      case 4:
        if (indef) { while (!at_break()) skip(); p++; } else for (uint64_t i = 0; i < arg; i++) skip();
        return;
      case 5:
        if (indef) { while (!at_break()) { skip(); skip(); } p++; } else for (uint64_t i = 0; i < arg; i++) { skip(); skip(); }
        return;
      case 6: skip(); return;
      default:  // 7: simple values and floats (their payload was consumed by head()); a stray break is malformed
        if (indef) bad("unexpected CBOR break");
        return;
    }
  }
  // containers: `open` returns the element count or ~0 for an indefinite one; `more` drives the loop for both forms
  uint64_t open(uint32_t want_major, const char* what) {
    skip_tags();
    uint32_t major; uint64_t arg; bool indef;
    head(major, arg, indef);
    if (major != want_major) bad(what);
    return indef ? ~0ull : arg;
  }
  bool more(uint64_t& left) {
    if (left == ~0ull) { if (at_break()) { p++; return false; } return true; }
    if (left == 0) return false;
    left--;
    return true;
  }
  bool is_null() { skip_tags(); return p < end && (d[p] == 0xf6 || d[p] == 0xf7); }
  int64_t integer(const char* what) {
    skip_tags();
    uint32_t major; uint64_t arg; bool indef;
    head(major, arg, indef);
    if (major == 0 && arg <= (uint64_t)INT64_MAX) return (int64_t)arg;
    if (major == 1 && arg <= (uint64_t)INT64_MAX) return -1 - (int64_t)arg;
    bad(what);
  }
  bool boolean(const char* what) {
    skip_tags();
    const uint8_t b = byte();
    if (b == 0xf4) return false;
    if (b == 0xf5) return true;
    bad(what);
  }
  // definite text string, compared in place
  void text(const uint8_t*& s, size_t& n, const char* what) {
    skip_tags();
    uint32_t major; uint64_t arg; bool indef;
    head(major, arg, indef);
    if (major != 3 || indef) bad(what);
    s = take(arg);
    n = arg;
  }
  static bool eq(const uint8_t* s, size_t n, const char* lit) { return strlen(lit) == n && !memcmp(s, lit, n); }
  // field element: byte string of 32 canonical little-endian bytes (zokrates_field/src/lib.rs:547-560); the reference's
  // visitor also accepts a sequence of small integers (:585-596)
  void field(uint8_t out[32]) {
    skip_tags();
    uint32_t major; uint64_t arg; bool indef;
    head(major, arg, indef);
    if (major == 2 && !indef) {
      if (arg != 32) bad("field element is not a 32-byte string");
      memcpy(out, take(32), 32);
      return;
    }
    if (major == 4) {
      uint64_t left = indef ? ~0ull : arg;
      size_t k = 0;
      while (more(left)) {
        const int64_t v = integer("field element byte");
        if (k >= 32 || v < 0 || v > 255) bad("field element is not a 32-byte string");
        out[k++] = (uint8_t)v;
      }
      if (k != 32) bad("field element is not a 32-byte string");
      return;
    }
    bad("field element is not a 32-byte string");
  }
};

struct ProgTerm {
  int64_t var;
  uint8_t coeff[32];
};

// One parsed program: R1CS in ark order (what zkb_r1cs_load takes), directive tables, statement schedule.
struct ProgData {
  int curve = 0;
  uint64_t N = 0, ni = 0, nw = 0, m = 0, m_ext = 0;   // m_ext - m: variables that only directives touch (no R1CS column)
  uint32_t n_ret = 0;
  std::vector<int64_t> arg_ids;
  std::vector<uint8_t> arg_private;
  std::vector<uint32_t> arg_cols;
  std::vector<int64_t> var_of_col;                    // m_ext entries: IR variable id of every column
  // CSR matrices
  std::vector<uint64_t> rowptr[3];
  std::vector<uint32_t> col[3];
  std::vector<uint64_t> val[3];                       // 4 words per term, canonical
  // directives
  std::vector<uint32_t> d_kind, d_arg, d_in_ptr, d_out_ptr, d_out_cols;
  std::vector<uint32_t> lc_ptr, lc_col;               // input j: combinations 2j (left) and 2j+1 (right)
  std::vector<uint64_t> lc_val;
  uint32_t n_unsupported = 0;
  // statement order and the level schedule
  std::vector<uint32_t> stmts;
  std::vector<uint32_t> row_level_ptr, rows, out_var, dir_level_ptr, dirs;   // level l: rows[row_level_ptr[l] ..), dirs[dir_level_ptr[l] ..)
  uint32_t n_levels = 0;
  std::vector<uint8_t> defined;                       // per column: some statement (or an input) gives it a value
  std::string schedule_error;                         // non-empty: the statements cannot be scheduled (compute-witness refuses)
  uint64_t r1cs = 0;                                  // handle of the loaded matrices
  mutable std::unordered_map<int64_t, uint32_t> col_of_var;   // IR variable id -> R1CS column, built on the first witness_parse
};

namespace prog_detail {

static const uint8_t CURVE_ID[3][4] = {{0xb4, 0xf7, 0xb5, 0xbd}, {0x40, 0xd8, 0xc1, 0xf9},   // zokrates_field/src/lib.rs:283-293
                                      {0xc2, 0x95, 0x5a, 0xb5}};                              // bn128, bls12_381, bls12_377

inline uint32_t le32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
inline uint64_t le64(const uint8_t* p) { return (uint64_t)le32(p) | (uint64_t)le32(p + 4) << 32; }

inline bool canonical(const uint8_t v[32], const uint32_t mod[8]) {   // v < modulus
  for (int i = 7; i >= 0; i--) {
    const uint32_t w = le32(v + 4 * i);
    if (w != mod[i]) return w < mod[i];
  }
  return false;
}

inline int64_t variable(Cbor& c) {   // Variable { id: isize }  (common/flat/variable.rs:6-12)
  uint64_t left = c.open(5, "Variable is not a map");
  int64_t id = 0;
  bool seen = false;
  while (c.more(left)) {
    const uint8_t* k; size_t n;
    c.text(k, n, "Variable key");
    if (Cbor::eq(k, n, "id")) { id = c.integer("Variable id"); seen = true; } else c.skip();
  }
  if (!seen) Cbor::bad("Variable without id");
  return id;
}

inline void lincomb(Cbor& c, const uint32_t mod[8], std::vector<ProgTerm>& out) {   // LinComb { span, value: Vec<(Variable, T)> }
  uint64_t left = c.open(5, "LinComb is not a map");
  bool seen = false;
  while (c.more(left)) {
    const uint8_t* k; size_t n;
    c.text(k, n, "LinComb key");
    if (!Cbor::eq(k, n, "value")) { c.skip(); continue; }
    seen = true;
    uint64_t terms = c.open(4, "LinComb value is not a sequence");
    while (c.more(terms)) {
      uint64_t pair = c.open(4, "LinComb term is not a pair");
      ProgTerm t;
      if (!c.more(pair)) Cbor::bad("LinComb term is not a pair");
      t.var = variable(c);
      if (!c.more(pair)) Cbor::bad("LinComb term is not a pair");
      c.field(t.coeff);
      if (c.more(pair)) Cbor::bad("LinComb term is not a pair");
      if (!canonical(t.coeff, mod)) Cbor::bad("non-canonical field element");
      out.push_back(t);
    }
  }
  if (!seen) Cbor::bad("LinComb without value");
}

inline void quadcomb(Cbor& c, const uint32_t mod[8], std::vector<ProgTerm>& l, std::vector<ProgTerm>& r) {
  uint64_t left = c.open(5, "QuadComb is not a map");
  bool sl = false, sr = false;
  while (c.more(left)) {
    const uint8_t* k; size_t n;
    c.text(k, n, "QuadComb key");
    if (Cbor::eq(k, n, "left")) { lincomb(c, mod, l); sl = true; }
    else if (Cbor::eq(k, n, "right")) { lincomb(c, mod, r); sr = true; }
    else c.skip();
  }
  if (!sl || !sr) Cbor::bad("QuadComb without left / right");
}

struct SolverRef { uint32_t kind; uint32_t arg; int64_t ref; };   // ref >= 0: index into the solvers section

inline SolverRef solver(Cbor& c) {
  c.skip_tags();
  SolverRef s{SOLVER_UNSUPPORTED, 0, -1};
  auto by_name = [&](const uint8_t* k, size_t n) -> uint32_t {
    if (Cbor::eq(k, n, "ConditionEq")) return SOLVER_CONDITION_EQ;
    if (Cbor::eq(k, n, "Bits")) return SOLVER_BITS;
    if (Cbor::eq(k, n, "Div")) return SOLVER_DIV;
    if (Cbor::eq(k, n, "Xor")) return SOLVER_XOR;
    if (Cbor::eq(k, n, "Or")) return SOLVER_OR;
    if (Cbor::eq(k, n, "ShaAndXorAndXorAnd")) return SOLVER_SHA_AXXA;
    if (Cbor::eq(k, n, "ShaCh")) return SOLVER_SHA_CH;
    if (Cbor::eq(k, n, "EuclideanDiv")) return SOLVER_EUCLIDEAN_DIV;
    return SOLVER_UNSUPPORTED;
  };
  if (c.p < c.end && (c.d[c.p] >> 5) == 3) {   // unit variant: text
    const uint8_t* k; size_t n;
    c.text(k, n, "Solver");
    s.kind = by_name(k, n);
    return s;
  }
  uint64_t left = c.open(5, "malformed Solver");
  if (!c.more(left)) Cbor::bad("malformed Solver");
  const uint8_t* k; size_t n;
  c.text(k, n, "Solver variant");
  if (Cbor::eq(k, n, "Bits")) {
    const int64_t w = c.integer("Bits width");
    if (w < 0 || w > 4096) Cbor::bad("Bits width");
    s.kind = SOLVER_BITS; s.arg = (uint32_t)w;
  } else if (Cbor::eq(k, n, "Ref")) {    // SolverIndexer replaced the solver by its index (serialize.rs:211-228)
    uint64_t rl = c.open(5, "RefCall is not a map");
    while (c.more(rl)) {
      const uint8_t* rk; size_t rn;
      c.text(rk, rn, "RefCall key");
      if (Cbor::eq(rk, rn, "index")) s.ref = c.integer("RefCall index"); else c.skip();
    }
    if (s.ref < 0) Cbor::bad("RefCall without index");
  } else {
    c.skip();                            // Zir(function), SnarkVerifyBls12377(n): no device path
  }
  if (c.more(left)) Cbor::bad("malformed Solver");
  return s;
}

}  // namespace prog_detail

// `out` bytes -> ProgData (matrices in ark order, directive tables, statement order).  `mod`: the scalar-field modulus.
inline void prog_parse(const uint8_t* data, size_t len, int curve, const uint32_t mod[8], ProgData& P) {
  using namespace prog_detail;
  if (len < 100) Cbor::bad("Invalid header");
  if (memcmp(data, "ZOK\0", 4)) Cbor::bad("Invalid magic number");
  const uint8_t version[4] = {3, 0, 0, 0};
  if (memcmp(data + 4, version, 4)) Cbor::bad("Invalid file version");
  if (memcmp(data + 8, CURVE_ID[curve], 4)) Cbor::bad("the program was compiled for another curve");
  const uint32_t n_cons = le32(data + 12);
  P.curve = curve;
  P.n_ret = le32(data + 16);
  uint64_t off[4], ln[4];
  for (int k = 0; k < 4; k++) {
    const uint32_t ty = le32(data + 20 + 20 * k);
    off[k] = le64(data + 24 + 20 * k);
    ln[k] = le64(data + 32 + 20 * k);
    if (ty < 1 || ty > 4) Cbor::bad("invalid section type");
    if (off[k] > len || ln[k] > len - off[k]) Cbor::bad("section out of bounds");
  }
  // parameters: Vec<Parameter { span, id: Variable, private: bool }>  (common/flat/parameter.rs:9-16)
  {
    Cbor c{data, (size_t)off[0], (size_t)(off[0] + ln[0])};
    uint64_t left = c.open(4, "Cannot read parameters");
    while (c.more(left)) {
      uint64_t f = c.open(5, "Cannot read parameters");
      int64_t id = 0; bool priv = false, si = false, sp = false;
      while (c.more(f)) {
        const uint8_t* k; size_t n;
        c.text(k, n, "Parameter key");
        if (Cbor::eq(k, n, "id")) { id = variable(c); si = true; }
        else if (Cbor::eq(k, n, "private")) { priv = c.boolean("Parameter private"); sp = true; }
        else c.skip();
      }
      if (!si || !sp) Cbor::bad("Cannot read parameters");
      P.arg_ids.push_back(id);
      P.arg_private.push_back(priv ? 1 : 0);
    }
  }
  // solvers: Vec<Solver>
  std::vector<SolverRef> table;
  if (ln[2]) {
    Cbor c{data, (size_t)off[2], (size_t)(off[2] + ln[2])};
    uint64_t left = c.open(4, "Cannot read solvers");
    while (c.more(left)) table.push_back(solver(c));
  }
  // ark symbol table: instance / witness numbering in allocation order (zokrates_ark/src/lib.rs:47-73,94-113)
  static constexpr uint32_t WIT = 0x80000000u;   // symbol = index | WIT for witness variables
  // Symbol table.  The compiler numbers its variables densely (ids 0 .. #variables, outputs -1, -2, ..), so non-negative ids
  // below a bound proportional to the file size live in a direct-index vector (one load instead of a hash lookup per term:
  // the parse of a 2^20-constraint program went from 0.72 s to the number in DESIGN.md §7); anything else goes to the map.
  struct SymTab {
    enum : uint32_t { UNSET = 0xFFFFFFFFu };
    std::vector<uint32_t> dense;
    std::unordered_map<int64_t, uint32_t> sparse;
    int64_t dense_cap = 0;
    uint32_t* find(int64_t id) {
      if (id >= 0 && id < dense_cap) {
        if ((size_t)id >= dense.size()) return nullptr;
        return dense[(size_t)id] == UNSET ? nullptr : &dense[(size_t)id];
      }
      auto it = sparse.find(id);
      return it == sparse.end() ? nullptr : &it->second;
    }
    void set(int64_t id, uint32_t v) {
      if (id >= 0 && id < dense_cap) {
        if ((size_t)id >= dense.size()) dense.resize(std::max<size_t>((size_t)id + 1, dense.size() * 2), UNSET);
        dense[(size_t)id] = v;
      } else {
        sparse[id] = v;
      }
    }
    bool count(int64_t id) { return find(id) != nullptr; }
  } sym;
  sym.dense_cap = (int64_t)std::min<size_t>(len / 8 + 1024, (size_t)1 << 28);   // a variable that occurs costs >= 8 bytes of file
  std::vector<int64_t> inst, wit;
  sym.set(0, 0);
  inst.push_back(0);
  for (size_t i = 0; i < P.arg_ids.size(); i++) {
    const int64_t id = P.arg_ids[i];
    if (sym.count(id)) Cbor::bad("duplicate argument");
    if (P.arg_private[i]) { sym.set(id, (uint32_t)wit.size() | WIT); wit.push_back(id); }
    else { sym.set(id, (uint32_t)inst.size()); inst.push_back(id); }
  }
  std::vector<uint32_t> rsym[3];          // per matrix: symbol of every term (columns are fixed once ni is known)
  for (int k = 0; k < 3; k++) { P.rowptr[k].reserve(std::min<size_t>((size_t)n_cons, len / 40) + 1); P.rowptr[k].push_back(0); }
  auto add_comb = [&](int k, const std::vector<ProgTerm>& terms) {
    for (const ProgTerm& t : terms) {
      const uint32_t* it = sym.find(t.var);
      uint32_t s;
      if (!it) {
        if (t.var < 0) { s = (uint32_t)inst.size(); inst.push_back(t.var); }
        else { s = (uint32_t)wit.size() | WIT; wit.push_back(t.var); }
        if (inst.size() >= 0x40000000u || wit.size() >= 0x40000000u) Cbor::bad("too many variables");
        sym.set(t.var, s);
      } else {
        s = *it;
      }
      rsym[k].push_back(s);
      for (int w = 0; w < 4; w++) P.val[k].push_back(le64(t.coeff + 8 * w));
    }
    P.rowptr[k].push_back(rsym[k].size());
  };
  // directive terms keep IR ids until every constraint has been seen (a directive does not allocate ark variables)
  std::vector<int64_t> lc_var, d_out_var;
  P.d_in_ptr.push_back(0); P.d_out_ptr.push_back(0); P.lc_ptr.push_back(0);
  std::vector<ProgTerm> tl, tr, tc;
  {
    Cbor c{data, (size_t)off[1], (size_t)(off[1] + ln[1])};
    while (c.p < c.end) {
      uint64_t one = c.open(5, "a Statement must be a one-entry map");
      if (!c.more(one)) Cbor::bad("a Statement must be a one-entry map");
      const uint8_t* k; size_t n;
      c.text(k, n, "Statement variant");
      if (Cbor::eq(k, n, "Constraint")) {
        tl.clear(); tr.clear(); tc.clear();
        uint64_t f = c.open(5, "ConstraintStatement is not a map");
        bool sq = false, sl = false;
        while (c.more(f)) {
          const uint8_t* fk; size_t fn;
          c.text(fk, fn, "ConstraintStatement key");
          if (Cbor::eq(fk, fn, "quad")) { quadcomb(c, mod, tl, tr); sq = true; }
          else if (Cbor::eq(fk, fn, "lin")) { lincomb(c, mod, tc); sl = true; }
          else c.skip();   // span, error
        }
        if (!sq || !sl) Cbor::bad("ConstraintStatement without quad / lin");
        if (P.rowptr[0].size() - 1 >= 0x7fffffffu) Cbor::bad("too many constraints");
        P.stmts.push_back((uint32_t)(P.rowptr[0].size() - 1));
        add_comb(0, tl); add_comb(1, tr); add_comb(2, tc);
      } else if (Cbor::eq(k, n, "Directive")) {
        uint64_t f = c.open(5, "DirectiveStatement is not a map");
        SolverRef sv{SOLVER_UNSUPPORTED, 0, -1};
        const uint32_t d = (uint32_t)P.d_kind.size();
        bool si = false, so = false, ss = false;
        while (c.more(f)) {
          const uint8_t* fk; size_t fn;
          c.text(fk, fn, "DirectiveStatement key");
          if (Cbor::eq(fk, fn, "inputs")) {
            si = true;
            uint64_t ins = c.open(4, "directive inputs");
            while (c.more(ins)) {
              tl.clear(); tr.clear();
              quadcomb(c, mod, tl, tr);
              for (const std::vector<ProgTerm>* side : {&tl, &tr}) {
                for (const ProgTerm& t : *side) {
                  lc_var.push_back(t.var);
                  for (int w = 0; w < 4; w++) P.lc_val.push_back(le64(t.coeff + 8 * w));
                }
                P.lc_ptr.push_back((uint32_t)lc_var.size());
              }
            }
          } else if (Cbor::eq(fk, fn, "outputs")) {
            so = true;
            uint64_t outs = c.open(4, "directive outputs");
            while (c.more(outs)) d_out_var.push_back(variable(c));
          } else if (Cbor::eq(fk, fn, "solver")) {
            sv = solver(c); ss = true;
          } else {
            c.skip();
          }
        }
        if (!si || !so || !ss) Cbor::bad("DirectiveStatement without inputs / outputs / solver");
        if (sv.ref >= 0) {
          if ((uint64_t)sv.ref >= table.size()) Cbor::bad("solver index out of range");
          sv = table[(size_t)sv.ref];
          if (sv.ref >= 0) Cbor::bad("nested solver reference");
        }
        {  // Solver::get_signature (common/solvers.rs:47-63): the statement must carry exactly that many inputs and outputs
          const uint32_t n_in = (uint32_t)(P.lc_ptr.size() - 1) / 2 - P.d_in_ptr.back();
          const uint32_t n_out = (uint32_t)d_out_var.size() - P.d_out_ptr.back();
          uint32_t want_in = n_in, want_out = n_out;
          switch (sv.kind) {
            case SOLVER_CONDITION_EQ: want_in = 1; want_out = 2; break;
            case SOLVER_BITS: want_in = 1; want_out = sv.arg; break;
            case SOLVER_DIV: case SOLVER_XOR: case SOLVER_OR: want_in = 2; want_out = 1; break;
            case SOLVER_SHA_AXXA: case SOLVER_SHA_CH: want_in = 3; want_out = 1; break;
            case SOLVER_EUCLIDEAN_DIV: want_in = 2; want_out = 2; break;
            default: break;
          }
          if (n_in != want_in || n_out != want_out) Cbor::bad("directive does not match the signature of its solver");
        }
        P.d_kind.push_back(sv.kind); P.d_arg.push_back(sv.arg);
        P.d_in_ptr.push_back((uint32_t)(P.lc_ptr.size() - 1) / 2);
        P.d_out_ptr.push_back((uint32_t)d_out_var.size());
        if (sv.kind == SOLVER_UNSUPPORTED) P.n_unsupported++;
        P.stmts.push_back(d | PROG_DIRECTIVE);
      } else if (Cbor::eq(k, n, "Log")) {
        c.skip();
      } else {
        Cbor::bad("unknown Statement variant");
      }
      if (c.more(one)) Cbor::bad("a Statement must be a one-entry map");
    }
  }
  P.N = P.rowptr[0].size() - 1;
  if (P.N != n_cons) Cbor::bad("constraint count in the header does not match the constraints section");
  P.ni = inst.size(); P.nw = wit.size(); P.m = P.ni + P.nw;
  for (int k = 0; k < 3; k++) {
    P.col[k].resize(rsym[k].size());
    for (size_t i = 0; i < rsym[k].size(); i++)
      P.col[k][i] = (rsym[k][i] & WIT) ? (uint32_t)P.ni + (rsym[k][i] & ~WIT) : rsym[k][i];
  }
  P.var_of_col = inst;
  P.var_of_col.insert(P.var_of_col.end(), wit.begin(), wit.end());
  auto col_of = [&](int64_t v) -> uint32_t {
    const uint32_t* it = sym.find(v);
    if (!it) {   // only directives touch it: an extra column behind the R1CS ones
      const uint32_t cidx = (uint32_t)P.var_of_col.size();
      sym.set(v, cidx | 0x40000000u);
      P.var_of_col.push_back(v);
      return cidx;
    }
    const uint32_t s = *it;
    if (s & 0x40000000u) return s & ~0x40000000u;
    return (s & WIT) ? (uint32_t)P.ni + (s & ~WIT) : s;
  };
  // NB: extra columns are numbered from m upwards: the tag bit keeps them apart from ark symbols in `sym`
  P.lc_col.resize(lc_var.size());
  for (size_t i = 0; i < lc_var.size(); i++) P.lc_col[i] = col_of(lc_var[i]);
  P.d_out_cols.resize(d_out_var.size());
  for (size_t i = 0; i < d_out_var.size(); i++) P.d_out_cols[i] = col_of(d_out_var[i]);
  P.m_ext = P.var_of_col.size();
  if (P.m_ext >= 0x40000000u) Cbor::bad("too many variables");
  P.arg_cols.resize(P.arg_ids.size());
  for (size_t i = 0; i < P.arg_ids.size(); i++) P.arg_cols[i] = col_of(P.arg_ids[i]);
}

// Level schedule of the statements (same rule and tie order as the sequential interpreter, lib.rs:61-138): a constraint
// whose linear side is ONE variable with coefficient one that has no value yet assigns it; every other constraint is a
// check and needs all of its variables; a directive needs its inputs and defines its outputs.  level(statement) = 1 + the
// deepest level it reads.  A read of a variable that no earlier statement defined fails in the reference (unwrap on the
// lookup, :366-378): recorded in schedule_error, compute-witness then refuses the program.
inline void prog_schedule(ProgData& P) {
  static constexpr uint32_t UNDEF = 0xFFFFFFFFu, CHECK = 0xFFFFFFFFu;
  std::vector<uint32_t> level(P.m_ext, UNDEF);
  level[0] = 0;
  for (uint32_t c : P.arg_cols) level[c] = 0;
  const size_t S = P.stmts.size();
  std::vector<uint32_t> slevel(S, 0), sout(S, CHECK);
  uint32_t max_level = 0;
  auto fail = [&](size_t s, const char* what) {
    if (P.schedule_error.empty()) P.schedule_error = std::string("statement ") + std::to_string(s) + " " + what;
  };
  for (size_t s = 0; s < S && P.schedule_error.empty(); s++) {
    const uint32_t st = P.stmts[s];
    uint32_t base = 0;
    if (!(st & PROG_DIRECTIVE)) {
      const uint32_t k = st;
      for (int mtx = 0; mtx < 2; mtx++)
        for (uint64_t i = P.rowptr[mtx][k]; i < P.rowptr[mtx][k + 1]; i++) {
          const uint32_t l = level[P.col[mtx][i]];
          if (l == UNDEF) { fail(s, "reads a variable that has no value yet"); break; }
          base = std::max(base, l);
        }
      if (!P.schedule_error.empty()) break;
      const uint64_t c0 = P.rowptr[2][k], c1 = P.rowptr[2][k + 1];
      const bool one_coeff = c1 - c0 == 1 && P.val[2][4 * c0] == 1 && P.val[2][4 * c0 + 1] == 0 && P.val[2][4 * c0 + 2] == 0 &&
                             P.val[2][4 * c0 + 3] == 0;
      if (one_coeff && level[P.col[2][c0]] == UNDEF) {
        sout[s] = P.col[2][c0];
        level[P.col[2][c0]] = base + 1;
      } else {
        for (uint64_t i = c0; i < c1; i++) {
          const uint32_t l = level[P.col[2][i]];
          if (l == UNDEF) { fail(s, "reads a variable that has no value yet"); break; }
          base = std::max(base, l);
        }
      }
      slevel[s] = base + 1;
    } else {
      const uint32_t d = st & ~PROG_DIRECTIVE;
      for (uint32_t q = 2 * P.d_in_ptr[d]; q < 2 * P.d_in_ptr[d + 1]; q++)
        for (uint32_t i = P.lc_ptr[q]; i < P.lc_ptr[q + 1]; i++) {
          const uint32_t l = level[P.lc_col[i]];
          if (l == UNDEF) { fail(s, "reads a variable that has no value yet"); break; }
          base = std::max(base, l);
        }
      if (!P.schedule_error.empty()) break;
      for (uint32_t i = P.d_out_ptr[d]; i < P.d_out_ptr[d + 1]; i++) {
        if (level[P.d_out_cols[i]] != UNDEF) { fail(s, "redefines a variable (not in SSA form)"); break; }
        level[P.d_out_cols[i]] = base + 1;
      }
      slevel[s] = base + 1;
    }
    max_level = std::max(max_level, slevel[s]);
  }
  if (!P.schedule_error.empty()) return;
  P.defined.resize(P.m_ext);
  for (size_t c = 0; c < P.m_ext; c++) P.defined[c] = level[c] != UNDEF;
  P.n_levels = max_level;
  P.row_level_ptr.assign((size_t)max_level + 1, 0);
  P.dir_level_ptr.assign((size_t)max_level + 1, 0);
  for (size_t s = 0; s < S; s++) {
    if (P.stmts[s] & PROG_DIRECTIVE) P.dir_level_ptr[slevel[s]]++; else P.row_level_ptr[slevel[s]]++;
  }
  // counts of level l sit at index l (levels start at 1): prefix sums turn index l into the END of level l
  for (uint32_t l = 1; l <= max_level; l++) { P.row_level_ptr[l] += P.row_level_ptr[l - 1]; P.dir_level_ptr[l] += P.dir_level_ptr[l - 1]; }
  P.rows.resize(P.row_level_ptr[max_level]); P.out_var.resize(P.rows.size()); P.dirs.resize(P.dir_level_ptr[max_level]);
  std::vector<uint32_t> rcur(max_level + 1, 0), dcur(max_level + 1, 0);
  for (uint32_t l = 1; l <= max_level; l++) { rcur[l] = P.row_level_ptr[l - 1]; dcur[l] = P.dir_level_ptr[l - 1]; }
  for (size_t s = 0; s < S; s++) {
    const uint32_t l = slevel[s];
    if (P.stmts[s] & PROG_DIRECTIVE) P.dirs[dcur[l]++] = P.stmts[s] & ~PROG_DIRECTIVE;
    else { P.rows[rcur[l]] = P.stmts[s]; P.out_var[rcur[l]++] = sout[s]; }
  }
}

// witness file -> full assignment in column order (m entries x 4 words); every R1CS variable must be present
inline void witness_parse(const ProgData& P, const uint8_t* data, size_t len, const uint32_t mod[8], std::vector<uint64_t>& z) {
  using namespace prog_detail;
  auto bad = [](const char* w) { throw Error(ZKB_E_FORMAT, std::string("witness file: ") + w); };
  if (len < 8) bad("truncated");
  const uint64_t n = le64(data);
  if (n > (len - 8) / 40) bad("truncated");
  std::unordered_map<int64_t, uint32_t>& col = P.col_of_var;
  if (col.empty()) {
    col.reserve(P.m * 2);
    for (uint32_t c = 0; c < P.m; c++) col.emplace(P.var_of_col[c], c);
  }
  z.assign(P.m * 4, 0);
  std::vector<uint8_t> seen(P.m, 0);
  for (uint64_t i = 0; i < n; i++) {
    const uint8_t* rec = data + 8 + 40 * i;
    const int64_t id = (int64_t)le64(rec);
    if (!canonical(rec + 8, mod)) bad("non-canonical field element");
    auto it = col.find(id);
    if (it == col.end()) continue;   // a variable the constraints never mention
    for (int w = 0; w < 4; w++) z[4 * (size_t)it->second + w] = le64(rec + 8 + 8 * w);
    seen[it->second] = 1;
  }
  for (uint32_t c = 0; c < P.m; c++)
    if (!seen[c]) bad("a variable of the constraint system has no value (the reference panics on the same lookup)");
}

// full assignment (m_ext x 4 words, canonical) -> witness file bytes, BTreeMap order = ascending signed id
inline void witness_write(const ProgData& P, const uint64_t* z_ext, std::vector<uint8_t>& out) {
  const std::vector<uint8_t>& defined = P.defined;
  std::vector<uint32_t> order;
  order.reserve(P.m_ext);
  for (uint32_t c = 0; c < P.m_ext; c++) if (defined[c]) order.push_back(c);
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return P.var_of_col[a] < P.var_of_col[b]; });
  out.resize(8 + 40 * order.size());
  const uint64_t n = order.size();
  memcpy(out.data(), &n, 8);
  for (size_t i = 0; i < order.size(); i++) {
    uint8_t* rec = out.data() + 8 + 40 * i;
    const int64_t id = P.var_of_col[order[i]];
    memcpy(rec, &id, 8);
    memcpy(rec + 8, z_ext + 4 * (size_t)order[i], 32);
  }
}

}  // namespace zkb
