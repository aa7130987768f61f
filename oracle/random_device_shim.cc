// oracle/random_device_shim.cc -- TEST INFRASTRUCTURE ONLY.
// Linked into oracle/_ref/stochastic_mz_tree*.so (see build_stoch_ref.py): the Stochastic MuZero reference tree draws every
// chance outcome as std::discrete_distribution(priors)(std::mt19937(std::random_device{}())) (ctree_stochastic_muzero/lib/
// cnode.cpp:610-630), which no seed reproduces.  libstdc++'s <bits/random.h> defines random_device::operator() inline as
// `return this->_M_getval();`, and libstdc++.so exports std::random_device::_M_getval() (GLIBCXX_3.4.18): checked with
// g++ 13.3 / libstdc++ 13 (random.h:1679-1680; `nm -D libstdc++.so.6` lists _ZNSt13random_device9_M_getvalEv).  This
// definition, made hidden by the .hidden directive below (a visibility attribute on a member of the default-visibility class
// is ignored; the linker keeps the most constraining visibility any object gives a symbol), binds the module's own calls at
// link time: nothing is exported, every other user of random_device is untouched, and each draw seeds std::mt19937 with the
// value the test sets.  The constructor and destructor stay libstdc++'s.
#include <random>

static unsigned int g_value = 0;

extern "C" __attribute__((visibility("default"))) void lz_oracle_set_random_device(unsigned int value) { g_value = value; }

__asm__(".hidden _ZNSt13random_device9_M_getvalEv");
std::random_device::result_type std::random_device::_M_getval() { return g_value; }
