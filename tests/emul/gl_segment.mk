# TEST-ONLY: host emulation of the genotyping segments (emul_gl_segment.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
libwhemul_gl_segment.so: emul_gl_segment.cpp $(C)/gl_pack.cpp $(C)/pack.cpp $(C)/hostpool.cpp $(wildcard $(C)/*.h)
	$(CXX) -std=c++17 -O2 -Wall -Wno-unknown-pragmas -fPIC -shared -pthread -o $@ emul_gl_segment.cpp $(C)/gl_pack.cpp $(C)/pack.cpp $(C)/hostpool.cpp
clean:
	rm -f libwhemul_gl_segment.so
