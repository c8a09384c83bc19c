// TEST INFRASTRUCTURE ONLY — declaration-only stand-in for htslib's kfunc.h (see ../README).
#ifndef REF_SHIM_VB_KFUNC_H
#define REF_SHIM_VB_KFUNC_H
double kt_fisher_exact(int n11, int n12, int n21, int n22, double* left, double* right, double* two);
#endif
