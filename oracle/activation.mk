# TEST INFRASTRUCTURE ONLY — builds liborc_activation.so, the CPU restatement of activatePointsMT's distance map and selection loop
# (orc_activation.cpp), with the reference's flags (CMakeLists.txt:L44-57: -O3, no -march).  `make -f activation.mk` from oracle/;
# __graft_entry__.build() runs it.
CXX ?= g++
CXXFLAGS = -O3 -std=c++17 -fPIC -Wall

all: liborc_activation.so

liborc_activation.so: orc_activation.cpp activation.mk
	$(CXX) $(CXXFLAGS) -shared -o $@ orc_activation.cpp

clean:
	rm -f liborc_activation.so
