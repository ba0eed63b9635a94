# TEST-ONLY: host emulation of whmec_haplotagphase (emul_haplotagphase.cpp).
CXX := /usr/bin/g++
C := ../../whatshap_b200/csrc
SRC := emul_haplotagphase.cpp $(C)/haplotagphase_plan.cpp
libwhemul_haplotagphase.so: $(SRC) $(C)/haplotagphase.h $(C)/haplotagphase_plan.h ../../include/whmec.h
	$(CXX) -std=c++17 -O2 -Wall -fPIC -shared -o $@ $(SRC)
clean:
	rm -f libwhemul_haplotagphase.so
