# TEST INFRASTRUCTURE ONLY — builds liborc_select.so, the CPU restatement of PixelSelector::makeMaps and makeNewTraces' loop (orc_select.cpp),
# with the reference's flags (CMakeLists.txt:L44-57: -O3, no -march).  `make -f select.mk` from oracle/; __graft_entry__.build() runs it.
CXX ?= g++
CXXFLAGS = -O3 -std=c++17 -fPIC -Wall

all: liborc_select.so

liborc_select.so: orc_select.cpp select.mk
	$(CXX) $(CXXFLAGS) -shared -o $@ orc_select.cpp

clean:
	rm -f liborc_select.so
