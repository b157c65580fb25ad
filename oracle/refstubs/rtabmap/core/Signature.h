// Stand-in for rtabmap/core/Signature.h: the reference's BayesFilter.cpp includes it but uses nothing from it.  TEST INFRASTRUCTURE ONLY.
#pragma once
