# oracle/geodetic.mk — builds _ref/libref_geodetic.so (TEST INFRASTRUCTURE, never linked by the product): the reference's own
# corelib/src/GeodeticCoords.cpp compiled against the stand-ins of refstubs/geodetic/ (cv::Point3d and friends) and wrapped by
# ref_geodetic.cpp, with the compiler flags of the other _ref libraries (Makefile).  Needs the reference's sources, so it runs where
# they are; the library travels with the tree.
#
#   make -f geodetic.mk
REF ?= /root/reference
CXX ?= g++
CXXFLAGS ?= -O2 -std=c++17 -fPIC -w -ffp-contract=off
GEOINC := -Irefstubs/geodetic -Irefstubs -I$(REF)/corelib/include

_ref/libref_geodetic.so: ref_geodetic.cpp refstubs/geodetic/opencv2/core/core.hpp
	mkdir -p _ref/obj/geodetic
	$(CXX) $(CXXFLAGS) $(GEOINC) -c $(REF)/corelib/src/GeodeticCoords.cpp -o _ref/obj/geodetic/GeodeticCoords.o
	$(CXX) $(CXXFLAGS) $(GEOINC) -c ref_geodetic.cpp -o _ref/obj/geodetic/ref_geodetic.o
	$(CXX) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -o $@ _ref/obj/geodetic/*.o
