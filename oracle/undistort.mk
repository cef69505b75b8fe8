# TEST INFRASTRUCTURE ONLY — builds liborc_undistort.so, the CPU restatement of Undistort::undistort<T> (orc_undistort.cpp), with the
# reference's flags (CMakeLists.txt:L44-57: -O3, no -march).  `make -f undistort.mk` from oracle/; __graft_entry__.build() runs it.
CXX ?= g++
CXXFLAGS = -O3 -std=c++17 -fPIC -Wall

all: liborc_undistort.so

liborc_undistort.so: orc_undistort.cpp undistort.mk
	$(CXX) $(CXXFLAGS) -shared -o $@ orc_undistort.cpp

clean:
	rm -f liborc_undistort.so
