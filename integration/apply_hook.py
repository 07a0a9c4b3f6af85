#!/usr/bin/env python3
"""Applies the in-extension hook of INTEGRATION.md (B) to a SCRATCH COPY of the reference.

    cp -r <reference source tree> /tmp/dthook
    python integration/apply_hook.py /tmp/dthook            # edits src/core/sort.cc and ci/ext.py
    (cd /tmp/dthook && python ci/ext.py build)              # the reference's own backend, ~2 min
    PYTHONPATH=/tmp/dthook/src python integration/check_hook.py

The script only INSERTS our own code next to short anchor strings; it carries no reference source.
What it adds:
  * src/core/sort.cc  -- `#include <dtb200.h>`, option `sort.b200` (bool, default False) and, inside
    `group()` just before the CPU SortContext is built, a call to `dtb_group` for material
    bool/int/float key columns whose outputs are wrapped exactly like get_result_rowindex() /
    extract_groups() do (sort.cc:596-616).  DTB_ENOTIMPL falls through to the CPU path (outside the
    named path); any other error is raised as a dt RuntimeError with dtb_last_error().
  * src/core/expr/fexpr_reduce_unary.cc -- option `sort.b200_reducers` (bool, default False; registered in
    sort.cc): sum/mean/min/max/count/countna of a plain numeric column of the frame go through
    `dtb_reduce` with the frame's RowIndex and the Groupby offsets, the result wrapped as a material
    column of the reference's output stype.  Anything else keeps the reference's own reducer columns.
  * src/core/column/view.{h,cc} -- `ArrayView_ColumnImpl<T>::materialize` override: with `sort.b200` on, a
    view of a material bool/int/float column through an ARR32/ARR64 RowIndex is gathered by `dtb_gather`
    (the generic path is a per-element virtual get_element loop, column_impl.cc:78-103).
  * src/core/expr/eval_context.cc -- a residency bracket (dtb_cache_begin/end) around EvalContext::evaluate():
    host columns staged by group() / the reducers / the gathers of one query are uploaded once.
  * ci/ext.py         -- include path of include/dtb200.h, link + rpath of datatable_b200/lib/libdtb200.so.
The reference's own tree is never touched.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

INCLUDE_ANCHOR = '#include "utils/misc.h"\n'
INCLUDE_ADD = '#include <dtb200.h>      // dtb200 engine C-ABI (drop-in for group()); -I<repo>/include, see ci/ext.py\n'

OPTION_ANCHOR = 'static bool sort_new = false;\n'
OPTION_ADD = ('static bool sort_b200 = false;   // option sort.b200: route group() through libdtb200\n'
              'bool dtb200_enabled() { return sort_b200; }\n'
              'static bool sort_b200_reducers = false;   // option sort.b200_reducers: reducers through dtb_reduce\n'
              'bool dtb200_reducers_enabled() { return sort_b200_reducers; }\n')

REGISTER_ANCHOR = '  dt::register_option(\n    "sort.new",'
REGISTER_ADD = '''  dt::register_option(
    "sort.b200",
    []{ return py::obool(sort_b200); },
    [](const py::Arg& value) {
      sort_b200 = value.to_bool_strict();
    },
    nullptr);

  dt::register_option(
    "sort.b200_reducers",
    []{ return py::obool(sort_b200_reducers); },
    [](const py::Arg& value) {
      sort_b200_reducers = value.to_bool_strict();
    },
    nullptr);

'''

HOOK_ANCHOR = '  bool do_groups = n > 1 || !(flags[0] & SortFlag::SORT_ONLY);\n  SortContext sc('
HOOK_ADD = '''  // ---- dtb200: the whole ordering + grouping on the GPU ---------------------------------
  if (sort_b200 && nrows <= 0x7FFFFFFFu) {
    bool eligible = true;
    std::vector<dtb_col> b200_keys(n);
    std::vector<int> b200_flags(n);
    for (size_t j = 0; j < n; ++j) {
      const Column& cj = columns[j];
      switch (cj.stype()) {
        case dt::SType::BOOL: case dt::SType::INT8: case dt::SType::INT16: case dt::SType::INT32:
        case dt::SType::INT64: case dt::SType::FLOAT32: case dt::SType::FLOAT64: break;
        default: eligible = false;
      }
      if (!eligible) break;
      b200_keys[j].data = cj.get_data_readonly();                 // material after the loop above
      b200_keys[j].stype = static_cast<int>(cj.stype());          // SType values == DtStype_* codes
      b200_keys[j].reserved = 0;
      b200_flags[j] = static_cast<int>(flags[j]) & (DTB_FLAG_DESCENDING | DTB_FLAG_SORT_ONLY);  // same bit values
    }
    if (eligible) {
      Buffer b200_order = Buffer::mem(nrows * sizeof(int32_t));
      Buffer b200_offsets = Buffer::mem((nrows + 1) * sizeof(int32_t));
      int64_t b200_ng = -1, b200_norder = 0;
      int rc = dtb_group(b200_keys.data(), static_cast<int>(n), b200_flags.data(),
                         static_cast<int>(na_pos),                // NaPosition FIRST/LAST/REMOVE = 1/2/3 = DTB_NA_*
                         static_cast<int64_t>(nrows), nullptr,
                         b200_order.xptr(), b200_offsets.xptr(), static_cast<int64_t>(nrows + 1),
                         &b200_ng, &b200_norder);
      if (rc == DTB_OK) {
        b200_order.resize(static_cast<size_t>(b200_norder) * sizeof(int32_t));
        result.first = RowIndex(std::move(b200_order), RowIndex::ARR32);
        if (b200_ng >= 0) {
          b200_offsets.resize(static_cast<size_t>(b200_ng + 1) * sizeof(int32_t));
          result.second = Groupby(static_cast<size_t>(b200_ng), std::move(b200_offsets));
        }
        return result;
      }
      if (rc != DTB_ENOTIMPL) {
        throw RuntimeError() << "dtb200: " << dtb_last_error();
      }
    }
  }

'''


# ---- reducers: src/core/expr/fexpr_reduce_unary.cc ---------------------------------------------------
RED_INCLUDE_ANCHOR = '#include "expr/workframe.h"\n'
RED_INCLUDE_ADD = '''#include <cstring>
#include "datatable.h"
#include "stype.h"
#include <dtb200.h>      // dtb200 engine C-ABI (reducers)
bool dtb200_reducers_enabled();   // sort.cc, option sort.b200_reducers
'''

RED_HELPER_ANCHOR = 'FExpr_ReduceUnary::FExpr_ReduceUnary(ptrExpr&& arg)'
RED_HELPER_ADD = '''// dtb200: reducer name -> DTB_OP_* (0 = not handled by the engine)
static int dtb200_op_of(const std::string& name) {
  if (name == "sum") return DTB_OP_SUM;
  if (name == "mean") return DTB_OP_MEAN;
  if (name == "min") return DTB_OP_MIN;
  if (name == "max") return DTB_OP_MAX;
  if (name == "count") return DTB_OP_COUNT;
  if (name == "countna") return DTB_OP_COUNTNA;
  return 0;
}

// dtb200: evaluate one reducer over a plain numeric column of frame `ifr` on the engine.
// Returns false when the case is outside the engine's scope (the caller keeps the CPU path).
static bool dtb200_reduce(EvalContext& ctx, size_t ifr, size_t icol, int op,
                          const Groupby& gby, Column* out)
{
  const Column& src = ctx.get_datatable(ifr)->get_column(icol);
  const RowIndex& ri = ctx.get_rowindex(ifr);
  if (src.is_virtual() || gby.size() == 0) return false;
  if (ri && !ri.isarr32()) return false;                       // ARR32 (the group() ordering) or identity
  switch (src.stype()) {
    case SType::BOOL: case SType::INT8: case SType::INT16: case SType::INT32:
    case SType::INT64: case SType::FLOAT32: case SType::FLOAT64: break;
    default: return false;
  }
  const int in_st = static_cast<int>(src.stype());             // SType values == DtStype_* codes
  const int out_st = dtb_reduce_out_stype(op, in_st);
  if (!out_st) return false;
  const size_t ng = gby.size();
  Buffer buf = Buffer::mem(ng * static_cast<size_t>(dtb_stype_size(out_st)));
  dtb_col v; v.data = src.get_data_readonly(); v.stype = in_st; v.reserved = 0;
  int rc = dtb_reduce(op, v, static_cast<int64_t>(src.nrows()),
                      ri ? static_cast<const void*>(ri.indices32()) : nullptr, 0,
                      gby.offsets_r(), static_cast<int64_t>(ng), nullptr, buf.xptr());
  if (rc == DTB_ENOTIMPL) return false;
  if (rc != DTB_OK) throw RuntimeError() << "dtb200: " << dtb_last_error();
  *out = Column::new_mbuf_column(ng, static_cast<SType>(out_st), std::move(buf));
  return true;
}


'''

RED_LOOP_ANCHOR = '    Column coli = wf.retrieve_column(i);\n    coli = evaluate1('
RED_LOOP_ADD = '''    {
      // dtb200: a plain numeric column of the frame, reduced by sum/mean/min/max/count on the engine
      size_t b200_ifr = 0, b200_icol = 0;
      const int b200_op = dtb200_reducers_enabled() ? dtb200_op_of(name()) : 0;
      if (b200_op && !is_wf_grouped && wf.is_reference_column(i, &b200_ifr, &b200_icol)) {
        Column b200_out;
        if (dtb200_reduce(ctx, b200_ifr, b200_icol, b200_op, gby, &b200_out)) {
          outputs.add_column(std::move(b200_out), wf.retrieve_name(i), Grouping::GtoONE);
          continue;
        }
      }
    }
'''

# ---- ArrayView gather: src/core/column/view.{h,cc} --------------------------------------------------------
VIEW_H_ANCHOR = '    // defined in sort.cc\n    void sort_grouped(const Groupby& gby, Column& out) override;\n'
VIEW_H_ADD = '    void materialize(Column& out, bool to_memory) override;   // dtb200: gather on the engine\n'

VIEW_CC_INCLUDE_ANCHOR = '#include "column/view.h"\n'
VIEW_CC_INCLUDE_ADD = '''#include "stype.h"
#include <dtb200.h>      // dtb200 engine C-ABI (RowIndex gather)
bool dtb200_enabled();   // sort.cc, option sort.b200
'''

VIEW_CC_ANCHOR = 'template class ArrayView_ColumnImpl<int32_t>;\n'
VIEW_CC_ADD = '''// dtb200: out[i] = indices[i] < 0 ? NA : arg[indices[i]] as one dtb_gather instead of the generic
// per-element virtual loop (column_impl.cc:78-103).  Anything the engine does not cover keeps that loop.
template <typename T>
void ArrayView_ColumnImpl<T>::materialize(Column& out, bool to_memory) {
  bool eligible = dtb200_enabled() && !arg.is_virtual() && nrows_ > 0;
  if (eligible) {
    switch (arg.stype()) {
      case SType::BOOL: case SType::INT8: case SType::INT16: case SType::INT32: case SType::INT64:
      case SType::FLOAT32: case SType::FLOAT64: case SType::DATE32: case SType::TIME64: break;
      default: eligible = false;
    }
  }
  if (eligible) {
    const int st = static_cast<int>(arg.stype());               // SType values == DtStype_* codes
    Buffer buf = Buffer::mem(nrows_ * static_cast<size_t>(dtb_stype_size(st)));
    dtb_col src; src.data = arg.get_data_readonly(); src.stype = st; src.reserved = 0;
    int rc = dtb_gather(src, static_cast<int64_t>(arg.nrows()), indices, sizeof(T) == 8,
                        static_cast<int64_t>(nrows_), nullptr, buf.xptr());
    if (rc == DTB_OK) {
      out = Column::new_mbuf_column(nrows_, arg.stype(), std::move(buf));
      return;
    }
    if (rc != DTB_ENOTIMPL) throw RuntimeError() << "dtb200: " << dtb_last_error();
  }
  ColumnImpl::materialize(out, to_memory);
}

'''

# ---- residency bracket: src/core/expr/eval_context.cc ---------------------------------------------------
EVAL_INCLUDE_ANCHOR = '#include "expr/eval_context.h"\n'
EVAL_INCLUDE_ADD = '''#include <dtb200.h>      // dtb200 engine C-ABI (residency bracket)
namespace { struct Dtb200CacheScope { Dtb200CacheScope() { dtb_cache_begin(); } ~Dtb200CacheScope() { dtb_cache_end(); } }; }
'''
EVAL_ANCHOR = 'py::oobj EvalContext::evaluate() {\n'
EVAL_ADD = '  Dtb200CacheScope dtb200_cache_scope;   // host columns staged by the engine stay in HBM for this query\n'

EXT_ANCHOR = '            ext.compiler.add_linker_flag("-lstdc++")\n'
EXT_ADD = '''            # dtb200: dtb200 engine C-ABI
            ext.compiler.add_compiler_flag("-I{inc}")
            ext.compiler.add_linker_flag("-L{lib}", "-ldtb200", "-Wl,-rpath,{lib}")
'''


def insert(text, anchor, add, before, what):
    if add in text:
        return text                                          # already applied
    i = text.find(anchor)
    if i < 0:
        sys.exit(f"apply_hook: anchor for {what} not found -- is this the expected reference revision?")
    if text.find(anchor, i + 1) >= 0:
        sys.exit(f"apply_hook: anchor for {what} is not unique")
    at = i if before else i + len(anchor)
    return text[:at] + add + text[at:]


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    tree = os.path.realpath(sys.argv[1])
    src = os.path.realpath(os.environ.get("DATATABLE_REFERENCE_SRC") or os.path.join(os.path.dirname(ROOT), "reference"))
    if tree == src or tree.startswith(src + os.sep):
        sys.exit(f"apply_hook: refusing to modify the reference's source tree {src}; work on a scratch copy")
    sort_cc = os.path.join(tree, "src", "core", "sort.cc")
    s = open(sort_cc).read()
    s = insert(s, INCLUDE_ANCHOR, INCLUDE_ADD, before=False, what="include")
    s = insert(s, OPTION_ANCHOR, OPTION_ADD, before=False, what="option flag")
    s = insert(s, REGISTER_ANCHOR, REGISTER_ADD, before=True, what="option registration")
    s = insert(s, HOOK_ANCHOR, HOOK_ADD, before=True, what="group() hook")
    open(sort_cc, "w").write(s)
    red_cc = os.path.join(tree, "src", "core", "expr", "fexpr_reduce_unary.cc")
    r = open(red_cc).read()
    r = insert(r, RED_INCLUDE_ANCHOR, RED_INCLUDE_ADD, before=False, what="reducer includes")
    r = insert(r, RED_HELPER_ANCHOR, RED_HELPER_ADD, before=True, what="reducer helper")
    r = insert(r, RED_LOOP_ANCHOR, RED_LOOP_ADD, before=True, what="reducer loop hook")
    open(red_cc, "w").write(r)
    view_h = os.path.join(tree, "src", "core", "column", "view.h")
    h = open(view_h).read()
    h = insert(h, VIEW_H_ANCHOR, VIEW_H_ADD, before=False, what="ArrayView materialize declaration")
    open(view_h, "w").write(h)
    view_cc = os.path.join(tree, "src", "core", "column", "view.cc")
    v = open(view_cc).read()
    v = insert(v, VIEW_CC_INCLUDE_ANCHOR, VIEW_CC_INCLUDE_ADD, before=False, what="view.cc includes")
    v = insert(v, VIEW_CC_ANCHOR, VIEW_CC_ADD, before=True, what="ArrayView materialize")
    open(view_cc, "w").write(v)
    eval_cc = os.path.join(tree, "src", "core", "expr", "eval_context.cc")
    ev = open(eval_cc).read()
    ev = insert(ev, EVAL_INCLUDE_ANCHOR, EVAL_INCLUDE_ADD, before=False, what="eval_context includes")
    ev = insert(ev, EVAL_ANCHOR, EVAL_ADD, before=False, what="residency bracket")
    open(eval_cc, "w").write(ev)
    ext_py = os.path.join(tree, "ci", "ext.py")
    e = open(ext_py).read()
    add = EXT_ADD.format(inc=os.path.join(ROOT, "include"), lib=os.path.join(ROOT, "datatable_b200", "lib"))
    e = insert(e, EXT_ANCHOR, add, before=False, what="build flags")
    open(ext_py, "w").write(e)
    print("apply_hook: patched", sort_cc, red_cc, "and", ext_py)


if __name__ == "__main__":
    main()
