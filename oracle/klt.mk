# oracle/klt.mk -- builds the KLT oracle (test infrastructure only), beside the libraries of oracle/Makefile and with its
# flags:
#   libsvo_oracle_klt.so    svo_oracle_klt.cpp: the LK pyramid, its Scharr derivatives and the pyramidal Lucas-Kanade tracker
#                           of the two-view initialisation, restated with every termination decision reported
# The reference the oracle is compared against is OpenCV's own calcOpticalFlowPyrLK, called from Python (oracle/binding_klt.py).
# usage: make -C oracle -f klt.mk
CXX ?= g++
CXXFLAGS ?= -O3 -std=c++17 -fPIC -mfma -mavx2 -ffp-contract=off -fno-signed-zeros -fno-math-errno -pthread -Wall -Wno-unused-function
all: libsvo_oracle_klt.so
libsvo_oracle_klt.so: svo_oracle_klt.cpp
	$(CXX) $(CXXFLAGS) -shared -o $@ svo_oracle_klt.cpp
