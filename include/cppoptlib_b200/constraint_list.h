// cppoptlib_b200/constraint_list.h -- the constraint lists of
// ConstrainedOptimizationProblem<Objective, Equalities<C...>, Inequalities<C...>> (cppoptlib.h): the reference's
// std::vector<FunctionExpr> of equality / inequality constraints (function_problem.h:54-107) as compile-time lists of
// device functors.  A list is a plain aggregate (head, tail), so it is trivially copyable and travels to the kernels
// by value (std::tuple is not trivially copyable in libstdc++); the AL kernels pick constraint i of a list with
// cno::al_list_eval (csrc/cno_auglag.cuh).  Shared by host (g++) and device (nvcc) translation units.
#ifndef CPPOPTLIB_B200_CONSTRAINT_LIST_H_
#define CPPOPTLIB_B200_CONSTRAINT_LIST_H_

namespace cppoptlib {
namespace function {

// Kind 0: equality constraints c(x) == 0; kind 1: inequality constraints c(x) >= 0.
template <int Kind, class... C>
struct ConstraintList;
template <int Kind>
struct ConstraintList<Kind> {
  static constexpr int size = 0;
};
template <int Kind, class H, class... R>
struct ConstraintList<Kind, H, R...> {
  static constexpr int size = 1 + static_cast<int>(sizeof...(R));
  H head;
  ConstraintList<Kind, R...> tail;
};

template <class... C>
using Equalities = ConstraintList<0, C...>;
template <class... C>
using Inequalities = ConstraintList<1, C...>;

}  // namespace function
}  // namespace cppoptlib

#endif  // CPPOPTLIB_B200_CONSTRAINT_LIST_H_
