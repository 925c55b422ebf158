// TEST INFRASTRUCTURE - NOT PRODUCT CODE, never loaded by the package.
//
// tests/cpp/contacts_host.cpp with the dual-number CF instances writing the VALUE parts of the records (TDS_CF_DUAL_PART = v): the
// records of the fp64 dual-number step in fp64, whose inputs and intermediate state are not rounded to fp32 after loading, so that
// central differences at h = 1e-6 resolve the JVP of the same instance.  Nothing outside tests/ builds or loads it.
#define TDS_CF_DUAL_PART v
#include "contacts_host.cpp"
