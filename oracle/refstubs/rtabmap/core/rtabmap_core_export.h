// Stand-in for the CMake-generated export header of the reference's corelib.  TEST INFRASTRUCTURE ONLY.
#pragma once
#define RTABMAP_CORE_EXPORT
