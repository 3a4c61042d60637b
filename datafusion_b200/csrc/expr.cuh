// expr.cuh — PhysicalExpr::evaluate on device columns (defined in filter.cu), shared with the join filter.
#pragma once
#include "batch.cuh"

namespace dfgpu {

// an AND / OR whose RHS can raise an error (division, cast): the reference may skip or pre-select that RHS (check_short_circuit, binary.rs:1182)
struct ExprGuard { int op_idx, lhs_start, rhs_start, slot; bool is_and; };
struct ExprPlan {
  std::vector<dfgpu_expr_node> nodes;
  std::vector<int> in_type, out_type;
  int root_type = 0;
  std::vector<ExprGuard> guards;
  bool has_decimal = false;        // some node reads or produces a Decimal128: evaluated on the 128-bit stack (expr_dec.cuh)
  std::vector<int64_t> aux;        // per node: power-of-ten rescale exponents of decimal BINARY / CAST nodes
};
// type inference + validation of a post-order program against a schema; max_nodes: the evaluator's program size (EProgram holds 48)
ExprPlan plan_expr(const int32_t* schema_types, int n_cols, const dfgpu_expr_node* nodes, int n_nodes, int max_nodes = 48);

uint64_t literal_bits(const dfgpu_expr_node& nd);
// Per batch: which guards are active (the reference would not evaluate the RHS on every row).  Evaluates each guard's LHS over the batch
// (count of TRUE / NULL) exactly as BinaryExpr::evaluate does before deciding; returns per node the (g_and, g_or) slot masks.
std::vector<std::pair<uint16_t, uint16_t>> resolve_guards(dfgpu_ctx* ctx, const ExprPlan& plan, const std::vector<DCol>& cols, int64_t n);   // literal value as the interpreter's 64-bit stack payload

struct EProgram;
void bind_program(const ExprPlan& plan, const std::vector<DCol>& cols, EProgram* prog, const std::vector<std::pair<uint16_t, uint16_t>>* gmasks = nullptr);

struct EvalResult { DCol column; DevBuf select_words; };
// want_column: materialise the value column; want_select: selection words (valid AND true) for predicates
EvalResult evaluate_expr(dfgpu_ctx* ctx, const ExprPlan& plan, const std::vector<DCol>& cols, int64_t n, bool want_column, bool want_select);

}  // namespace dfgpu
