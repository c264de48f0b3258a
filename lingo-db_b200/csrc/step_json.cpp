// step_json.cpp — serialised execution steps: the descriptor a compiler hook hands to the GPU backend, as text.
//
// In the reference an execution step reaches the runtime as generated CODE plus small serialised descriptions
// (DataSource::get(VarLen32 description) deserialises a hex string, DataSourceIteration.cpp:57-88; handleExecutionStepCPU,
// SubOpToControlFlow.cpp:4363-4394).  The GPU backend receives DATA instead of code (include/ldb_gpu.h), so a step is fully
// described by a document: this file parses that document — JSON, optionally hex-encoded like the reference's
// serializeToHexString payloads — resolves table and state NAMES against the context's registries, creates the sink state when
// the step says so, and runs ldb_gpu_run_pipeline.  It is what `GPUPatternList` would emit per step (SURVEY §8 f1); the five
// TPC-H plans are kept as step lists under tests/golden/plans/ and run through it (tests/test_gpu_steps.py).
#include "context.h"

#include <cstdio>
#include <cstring>
#include <deque>
#include <map>
#include <memory>
#include <string>
#include <vector>

namespace {
// ---------------------------------------------------------------- a small JSON reader (objects, arrays, strings, integers, bools)
struct J {
   enum Kind { NUL, BOOL, INT, STR, ARR, OBJ } kind = NUL;
   bool b = false;
   int64_t i = 0;
   std::string s;
   std::vector<J> a;
   std::vector<std::pair<std::string, J>> o;
   const J* get(const char* k) const {
      for (auto& kv : o)
         if (kv.first == k) return &kv.second;
      return nullptr;
   }
};
struct Parser {
   const char* p;
   const char* end;
   [[noreturn]] void fail(const std::string& m) const { throw ldb::ApiError(LDB_ERR_INVALID, "step description: " + m); }
   void ws() {
      while (p < end && (*p == ' ' || *p == '\n' || *p == '\t' || *p == '\r')) p++;
   }
   J value() {
      ws();
      if (p >= end) fail("unexpected end");
      J j;
      if (*p == '{') {
         p++;
         j.kind = J::OBJ;
         ws();
         if (p < end && *p == '}') {
            p++;
            return j;
         }
         while (true) {
            ws();
            J k = value();
            if (k.kind != J::STR) fail("object key must be a string");
            ws();
            if (p >= end || *p != ':') fail("':' expected");
            p++;
            j.o.emplace_back(k.s, value());
            ws();
            if (p < end && *p == ',') {
               p++;
               continue;
            }
            if (p < end && *p == '}') {
               p++;
               return j;
            }
            fail("',' or '}' expected");
         }
      }
      if (*p == '[') {
         p++;
         j.kind = J::ARR;
         ws();
         if (p < end && *p == ']') {
            p++;
            return j;
         }
         while (true) {
            j.a.push_back(value());
            ws();
            if (p < end && *p == ',') {
               p++;
               continue;
            }
            if (p < end && *p == ']') {
               p++;
               return j;
            }
            fail("',' or ']' expected");
         }
      }
      if (*p == '"') {
         p++;
         j.kind = J::STR;
         while (p < end && *p != '"') {
            if (*p == '\\') {
               p++;
               if (p >= end) fail("bad escape");
               switch (*p) {
                  case 'n': j.s += '\n'; break;
                  case 't': j.s += '\t'; break;
                  case '"': j.s += '"'; break;
                  case '\\': j.s += '\\'; break;
                  case '/': j.s += '/'; break;
                  default: fail("unsupported escape");
               }
               p++;
            } else {
               j.s += *p++;
            }
         }
         if (p >= end) fail("unterminated string");
         p++;
         return j;
      }
      if (!strncmp(p, "true", 4) && end - p >= 4) {
         p += 4;
         j.kind = J::BOOL;
         j.b = true;
         return j;
      }
      if (!strncmp(p, "false", 5) && end - p >= 5) {
         p += 5;
         j.kind = J::BOOL;
         return j;
      }
      if (!strncmp(p, "null", 4) && end - p >= 4) {
         p += 4;
         return j;
      }
      if (*p == '-' || (*p >= '0' && *p <= '9')) {
         bool neg = *p == '-';
         if (neg) p++;
         if (p >= end || *p < '0' || *p > '9') fail("digit expected");
         int64_t v = 0;
         while (p < end && *p >= '0' && *p <= '9') v = v * 10 + (*p++ - '0');
         if (p < end && (*p == '.' || *p == 'e' || *p == 'E')) fail("numbers are integers (decimal constants travel as strings, like FilterDescription values)");
         j.kind = J::INT;
         j.i = neg ? -v : v;
         return j;
      }
      fail(std::string("unexpected character '") + *p + "'");
   }
};
J parseJson(const std::string& text) {
   Parser ps{text.data(), text.data() + text.size()};
   J j = ps.value();
   ps.ws();
   if (ps.p != ps.end) ps.fail("trailing characters");
   return j;
}
std::string str(const J& o, const char* k, bool required = true) {
   const J* v = o.get(k);
   if (!v || v->kind == J::NUL) {
      if (required) throw ldb::ApiError(LDB_ERR_INVALID, std::string("step description: missing \"") + k + "\"");
      return "";
   }
   if (v->kind != J::STR) throw ldb::ApiError(LDB_ERR_INVALID, std::string("step description: \"") + k + "\" must be a string");
   return v->s;
}
int64_t num(const J& o, const char* k, int64_t dflt) {
   const J* v = o.get(k);
   if (!v || v->kind == J::NUL) return dflt;
   if (v->kind == J::BOOL) return v->b;
   if (v->kind != J::INT) throw ldb::ApiError(LDB_ERR_INVALID, std::string("step description: \"") + k + "\" must be an integer");
   return v->i;
}
const std::vector<J>& arr(const J& o, const char* k) {
   static const std::vector<J> empty;
   const J* v = o.get(k);
   if (!v || v->kind == J::NUL) return empty;
   if (v->kind != J::ARR) throw ldb::ApiError(LDB_ERR_INVALID, std::string("step description: \"") + k + "\" must be an array");
   return v->a;
}
int lookup(const std::map<std::string, int>& m, const std::string& k, const char* what) {
   auto it = m.find(k);
   if (it == m.end()) throw ldb::ApiError(LDB_ERR_UNSUPPORTED, std::string("step description: unknown ") + what + " \"" + k + "\"");
   return it->second;
}
const std::map<std::string, int> kKinds = {{"scan_reduce", LDB_PIPE_SCAN_REDUCE}, {"scan_groupby", LDB_PIPE_SCAN_GROUPBY}, {"scan_build", LDB_PIPE_SCAN_BUILD},
                                           {"scan_probe_agg", LDB_PIPE_SCAN_PROBE_AGG}, {"scan_probe2_groupby", LDB_PIPE_SCAN_PROBE2_GROUPBY},
                                           {"scan_star_probe_groupby", LDB_PIPE_SCAN_STAR_PROBE_GROUPBY}};
const std::map<std::string, int> kOps = {{"=", LDB_EQ}, {"!=", LDB_NEQ}, {"<", LDB_LT}, {"<=", LDB_LTE}, {">", LDB_GT}, {">=", LDB_GTE}, {"notnull", LDB_NOTNULL}, {"in", LDB_IN}, {"contains", LDB_CONTAINS}};
const std::map<std::string, int> kExprs = {{"col", LDB_EXPR_COL}, {"mul", LDB_EXPR_MUL}, {"mul_1minus", LDB_EXPR_MUL_1MINUS}, {"mul_1minus_1plus", LDB_EXPR_MUL_1MINUS_1PLUS},
                                           {"one", LDB_EXPR_ONE}, {"mul_1minus_minus_paymul", LDB_EXPR_MUL_1MINUS_MINUS_PAYMUL}};

// the parsed step with everything a LdbPipelineDesc points to kept alive
struct Step {
   LdbPipelineDesc d{};
   std::deque<std::string> keep;
   std::vector<LdbFilterDesc> filters;
   std::string source, sinkName, sinkType;
   std::vector<std::string> probeNames;
   int64_t sinkExpected = 0;
   int32_t sinkNKeys = 0, sinkNAggs = 0, sinkCapacity = 64, sinkFlags = 0, sinkNSide = 0, sinkKeyMin = 0, sinkKeyMax = -1;
   bool sinkCreate = false;
   const char* own(const std::string& s) {
      keep.push_back(s);
      return keep.back().c_str();
   }
};
void parseStep(const J& j, Step& st) {
   if (j.kind != J::OBJ) throw ldb::ApiError(LDB_ERR_INVALID, "step description: an object is expected");
   LdbPipelineDesc& d = st.d;
   d.kind = lookup(kKinds, str(j, "kind"), "pipeline kind");
   st.source = str(j, "source");
   for (auto& f : arr(j, "filters")) {
      LdbFilterDesc fd{};
      fd.column = st.own(str(f, "column"));
      fd.op = lookup(kOps, str(f, "op"), "filter op");
      if (fd.op == LDB_IN) {
         auto& vals = arr(f, "values");
         if (vals.empty() || vals.size() > LDB_MAX_IN_VALUES) throw ldb::ApiError(LDB_ERR_UNSUPPORTED, "step description: IN lists hold 1..8 values");
         fd.n_values = (int32_t) vals.size();
         fd.value_is_int = vals[0].kind == J::INT;
         for (size_t k = 0; k < vals.size(); k++) {
            if (vals[k].kind == J::INT) fd.int_values[k] = vals[k].i;
            else if (vals[k].kind == J::STR) fd.str_values[k] = st.own(vals[k].s);
            else throw ldb::ApiError(LDB_ERR_INVALID, "step description: IN values are integers or strings");
         }
      } else if (fd.op != LDB_NOTNULL) {
         const J* v = f.get("value");
         if (!v) throw ldb::ApiError(LDB_ERR_INVALID, "step description: filter without \"value\"");
         if (v->kind == J::INT) {
            fd.value_is_int = 1;
            fd.int_value = v->i;
         } else if (v->kind == J::STR) {
            fd.str_value = st.own(v->s);
         } else {
            throw ldb::ApiError(LDB_ERR_INVALID, "step description: filter value must be an integer or a string");
         }
      }
      st.filters.push_back(fd);
   }
   d.n_filters = (int32_t) st.filters.size();
   auto& keys = arr(j, "keys");
   if (keys.size() > LDB_MAX_KEYS) throw ldb::ApiError(LDB_ERR_UNSUPPORTED, "step description: at most 2 group keys in a specialised pipeline");
   d.n_keys = (int32_t) keys.size();
   for (size_t k = 0; k < keys.size(); k++) d.key_columns[k] = st.own(keys[k].s);
   auto& aggs = arr(j, "aggs");
   if (aggs.size() > LDB_MAX_AGGS) throw ldb::ApiError(LDB_ERR_UNSUPPORTED, "step description: at most 8 aggregates");
   d.n_aggs = (int32_t) aggs.size();
   for (size_t a = 0; a < aggs.size(); a++) {
      d.aggs[a].expr = lookup(kExprs, str(aggs[a], "expr"), "aggregate expression");
      auto& cols = arr(aggs[a], "columns");
      if (cols.size() > 3) throw ldb::ApiError(LDB_ERR_INVALID, "step description: an aggregate has at most 3 operand columns");
      for (size_t c = 0; c < cols.size(); c++) d.aggs[a].columns[c] = st.own(cols[c].s);
   }
   auto& probes = arr(j, "probes");
   if (probes.size() > LDB_MAX_PROBES) throw ldb::ApiError(LDB_ERR_UNSUPPORTED, "step description: at most 3 probes");
   d.n_probes = (int32_t) probes.size();
   for (size_t k = 0; k < probes.size(); k++) {
      st.probeNames.push_back(str(probes[k], "state"));
      d.probe_key_columns[k] = st.own(str(probes[k], "key"));
      std::string k2 = str(probes[k], "key2", false);
      d.probe_key2_columns[k] = k2.empty() ? nullptr : st.own(k2);
   }
   if (const J* b = j.get("build")) {
      d.build_key_column = st.own(str(*b, "key"));
      std::string k2 = str(*b, "key2", false), pay = str(*b, "payload", false), pe = str(*b, "payload_expr", false);
      d.build_key2_column = k2.empty() ? nullptr : st.own(k2);
      d.build_payload_column = pay.empty() ? nullptr : st.own(pay);
      d.build_payload_expr = pe == "year" ? LDB_PAYLOAD_YEAR : LDB_PAYLOAD_COLUMN;
      auto& side = arr(*b, "side");
      if (side.size() > LDB_MAX_SIDE) throw ldb::ApiError(LDB_ERR_UNSUPPORTED, "step description: at most 2 side columns");
      d.n_side = (int32_t) side.size();
      for (size_t k = 0; k < side.size(); k++) d.side_columns[k] = st.own(side[k].s);
   }
   const J* sink = j.get("sink");
   if (!sink || sink->kind != J::OBJ) throw ldb::ApiError(LDB_ERR_INVALID, "step description: missing \"sink\"");
   st.sinkName = str(*sink, "name");
   if (const J* c = sink->get("create")) {
      st.sinkCreate = true;
      st.sinkType = str(*c, "type");
      st.sinkNKeys = (int32_t) num(*c, "n_keys", 0);
      st.sinkNAggs = (int32_t) num(*c, "n_aggs", 0);
      st.sinkCapacity = (int32_t) num(*c, "capacity", 64);
      st.sinkExpected = num(*c, "expected_rows", 1024);
      st.sinkFlags = (num(*c, "unique", 1) ? LDB_JOIN_UNIQUE : 0) | (num(*c, "no_bloom", 0) ? LDB_JOIN_NO_BLOOM : 0);
      st.sinkNSide = (int32_t) num(*c, "n_side", 0);
      st.sinkKeyMin = (int32_t) num(*c, "key_min", 0);
      st.sinkKeyMax = (int32_t) num(*c, "key_max", -1);
      static const char* types[] = {"simple", "groupby", "join", "join_pair", "join_direct"};
      bool ok = false;
      for (auto* t : types) ok |= st.sinkType == t;
      if (!ok) throw ldb::ApiError(LDB_ERR_UNSUPPORTED, "step description: unknown sink type \"" + st.sinkType + "\"");
   }
}
std::string fromHex(const char* hex) {
   const size_t n = strlen(hex);
   if (n % 2) throw ldb::ApiError(LDB_ERR_INVALID, "step description: odd number of hex digits");
   auto nib = [](char c) -> int {
      if (c >= '0' && c <= '9') return c - '0';
      if (c >= 'a' && c <= 'f') return c - 'a' + 10;
      if (c >= 'A' && c <= 'F') return c - 'A' + 10;
      throw ldb::ApiError(LDB_ERR_INVALID, "step description: not a hex digit");
   };
   std::string out(n / 2, '\0');
   for (size_t i = 0; i < n / 2; i++) out[i] = (char) (nib(hex[2 * i]) * 16 + nib(hex[2 * i + 1]));
   return out;
}
void check(int rc, const LdbError& e) {
   if (rc != LDB_OK) throw ldb::ApiError(rc, e.message);
}
} // namespace

extern "C" {

// structure check only — no device needed (the compiler side can validate what it emits)
int ldb_gpu_step_validate(const char* json, LdbError* err) {
   return ldb::guarded(err, [&] {
      if (!json) throw ldb::ApiError(LDB_ERR_INVALID, "null argument");
      Step st;
      parseStep(parseJson(json), st);
   });
}
// name → handle registries of the context (states a step created or the caller registered)
int ldb_gpu_register_state(LdbContext* ctx, const char* name, LdbState* s, LdbError* err) {
   return ldb::guarded(err, [&] {
      if (!ctx || !name || !s) throw ldb::ApiError(LDB_ERR_INVALID, "null argument");
      ctx->namedStates[name] = s;
   });
}
LdbState* ldb_gpu_find_state(LdbContext* ctx, const char* name) {
   if (!ctx || !name) return nullptr;
   auto it = ctx->namedStates.find(name);
   return it == ctx->namedStates.end() ? nullptr : it->second;
}
int ldb_gpu_run_step(LdbContext* ctx, const char* json, LdbError* err) {
   return ldb::guarded(err, [&] {
      if (!ctx || !json) throw ldb::ApiError(LDB_ERR_INVALID, "null argument");
      Step st;
      parseStep(parseJson(json), st);
      LdbPipelineDesc& d = st.d;
      d.filters = st.filters.data();
      for (LdbTable* t : ctx->tables) // the most recently created table of that name
         if (t->name == st.source) d.source = t;
      if (!d.source) throw ldb::ApiError(LDB_ERR_INVALID, "step description: no table named \"" + st.source + "\" in this context");
      for (size_t k = 0; k < st.probeNames.size(); k++) {
         d.probe_states[k] = ldb_gpu_find_state(ctx, st.probeNames[k].c_str());
         if (!d.probe_states[k]) throw ldb::ApiError(LDB_ERR_INVALID, "step description: no state named \"" + st.probeNames[k] + "\"");
      }
      LdbError e;
      LdbState* sink = ldb_gpu_find_state(ctx, st.sinkName.c_str());
      if (st.sinkCreate) {
         if (st.sinkType == "simple") check(ldb_gpu_simple_state_create(ctx, st.sinkNAggs, &sink, &e), e);
         else if (st.sinkType == "groupby") check(ldb_gpu_groupby_create(ctx, st.sinkNKeys, st.sinkNAggs, st.sinkCapacity, &sink, &e), e);
         else if (st.sinkType == "join") check(ldb_gpu_join_table_create(ctx, st.sinkExpected, st.sinkFlags, st.sinkNSide, st.sinkNAggs, &sink, &e), e);
         else if (st.sinkType == "join_pair") check(ldb_gpu_join_table_create_pair(ctx, st.sinkExpected, st.sinkFlags, &sink, &e), e);
         else check(ldb_gpu_join_table_create_direct(ctx, st.sinkKeyMin, st.sinkKeyMax, &sink, &e), e);
         ctx->namedStates[st.sinkName] = sink;
      }
      if (!sink) throw ldb::ApiError(LDB_ERR_INVALID, "step description: no state named \"" + st.sinkName + "\" (add \"create\")");
      d.sink = sink;
      check(ldb_gpu_run_pipeline(ctx, &d, &e), e);
   });
}
// the same document hex-encoded, as the reference ships its serialised descriptions (utility::serializeToHexString →
// DataSource::get, DataSourceIteration.cpp:57-88)
int ldb_gpu_run_step_hex(LdbContext* ctx, const char* hex, LdbError* err) {
   return ldb::guarded(err, [&] {
      if (!hex) throw ldb::ApiError(LDB_ERR_INVALID, "null argument");
      const std::string json = fromHex(hex);
      LdbError e;
      check(ldb_gpu_run_step(ctx, json.c_str(), &e), e);
   });
}

} // extern "C"
