#include "bitnetmcu_b200.h" /* the reference-named symbols of the library (section 1), replacing the reference kernels */
