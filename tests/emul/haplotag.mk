# TEST-ONLY: host emulation of whmec_haplotag (emul_haplotag.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_haplotag.cpp $(C)/haplotag_plan.cpp
libwhemul_haplotag.so: $(SRC) $(C)/haplotag.h $(C)/haplotag_plan.h ../../include/whmec.h
	$(CXX) -std=c++17 -O2 -Wall -fPIC -shared -o $@ $(SRC)
clean:
	rm -f libwhemul_haplotag.so
