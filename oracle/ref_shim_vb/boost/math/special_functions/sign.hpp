// TEST INFRASTRUCTURE ONLY — declaration-only stand-in (see ref_shim_vb/README); the VB path never calls these.
#include "../decls.hpp"
