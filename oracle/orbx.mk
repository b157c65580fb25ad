# oracle/orbx.mk — builds _ref/libref_orbx.so (TEST INFRASTRUCTURE, never linked by the product): the reference's own
# corelib/src/opencv/ORBextractor.cc compiled against the OpenCV stand-ins of refstubs/orbx/ (types real, image operations aborting)
# and wrapped by ref_orbx.cpp, with the compiler flags of the other _ref libraries (Makefile).  Needs the reference's sources, so it
# runs where they are; the library travels with the tree.
#
#   make -f orbx.mk
REF ?= /root/reference
CXX ?= g++
CXXFLAGS ?= -O2 -std=c++17 -fPIC -w -ffp-contract=off
ORBXINC := -Irefstubs/orbx -I$(REF)/corelib/src/opencv

_ref/libref_orbx.so: ref_orbx.cpp $(wildcard refstubs/orbx/opencv2/*/*)
	mkdir -p _ref/obj/orbx
	$(CXX) $(CXXFLAGS) $(ORBXINC) -c $(REF)/corelib/src/opencv/ORBextractor.cc -o _ref/obj/orbx/ORBextractor.o
	$(CXX) $(CXXFLAGS) $(ORBXINC) -c ref_orbx.cpp -o _ref/obj/orbx/ref_orbx.o
	$(CXX) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL -o $@ _ref/obj/orbx/*.o
