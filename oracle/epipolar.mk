# oracle/epipolar.mk -- builds the epipolar-options oracle and its reference wrapper (test infrastructure only), beside the
# libraries of oracle/Makefile and with its flags:
#   libsvo_oracle_epipolar.so    svo_oracle_epipolar.cpp (the oracle of svo_oracle.cpp plus findEpipolarMatchDirect and
#                                DepthFilter::updateSeeds under every Matcher::Options setting)
#   _ref/libsvo_ref_epipolar.so  ref_wrap_epipolar.cpp with the reference's own sources, against the stand-in headers of shim/
#                                (built only where the reference exists; the tests replay its recorded outputs elsewhere)
# usage: make -C oracle -f epipolar.mk [ref]
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -mfma -mavx2 -ffp-contract=off -fno-signed-zeros -fno-math-errno -pthread -Wall -Wno-unused-function
all: libsvo_oracle_epipolar.so
libsvo_oracle_epipolar.so: svo_oracle_epipolar.cpp svo_oracle.cpp svo_oracle_align.inc svo_oracle_depth.inc svo_oracle_pose.inc svo_oracle_reproject.inc svo_oracle_detect.inc fast_ext.h oracle_math.h svo_oracle.h
	$(CXX) $(CXXFLAGS) -shared -o $@ svo_oracle_epipolar.cpp

REF ?= /root/reference
REF_SRCS = feature_alignment sparse_img_align matcher pose_optimizer point depth_filter feature_detection reprojector map config frame
_ref/libsvo_ref_epipolar.so: ref_wrap_epipolar.cpp ref_wrap.cpp ref_wrap_reproject.cpp svo_oracle.h fast_ext.h $(wildcard shim/*/*) oracle_math.h
	mkdir -p _ref
	$(CXX) -O3 -std=c++17 -fPIC -mfma -mavx2 -msse2 -fno-signed-zeros -fno-math-errno -funroll-loops -w \
	  -I shim -I $(REF)/svo/include -pthread -shared -o $@ ref_wrap_epipolar.cpp ref_wrap_reproject.cpp $(addprefix $(REF)/svo/src/,$(addsuffix .cpp,$(REF_SRCS)))
ref: _ref/libsvo_ref_epipolar.so
