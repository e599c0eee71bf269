// k_expr_text.cu -- vm_kernel<true, true>: the expression VM of the programs that cast floats or decimals to text or parse floats
// or booleans from it (float_text.cuh).  A module of its own, so that its out-of-line calls leave the register allocation of the
// other instantiations in k_expr.cu alone.
#define AURON_VM_TEXT_TU
#include "k_expr.cu"
