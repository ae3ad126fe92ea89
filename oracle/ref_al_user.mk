# oracle/ref_al_user.mk -- builds _ref/libcno_ref_al_user.so from ref_al_user.cc: the reference's own AugmentedLagrangian,
# functors and operators on the functor-constrained test problems (test infrastructure, not product).  Same flags and
# shim as _ref/libcno_ref.so in Makefile; only built when $(REFERENCE) exists.
#   make -C oracle -f ref_al_user.mk REFERENCE=<reference tree>
REFERENCE ?= /root/reference
CXX = g++
CXXFLAGS = -O2 -ffp-contract=off -fno-fast-math -fPIC -fopenmp -std=c++17 -Wall

all:
	@if [ -d "$(REFERENCE)/include/cppoptlib" ]; then $(MAKE) -f ref_al_user.mk _ref/libcno_ref_al_user.so; \
	else echo "reference tree absent: keeping prebuilt oracle/_ref/libcno_ref_al_user.so (if any)"; fi

_ref/libcno_ref_al_user.so: ref_al_user.cc ref_shim/Eigen/Core ref_shim/Eigen/Dense cno_oracle.h cno_al_oracle.h ../include/cno.h ../include/cno_al.h
	$(MAKE) libcno_oracle.so
	mkdir -p _ref
	$(CXX) $(CXXFLAGS) -shared -o $@ ref_al_user.cc -Iref_shim -I$(REFERENCE)/include -L. -lcno_oracle -Wl,-rpath,'$$ORIGIN/..'

.PHONY: all
