// Test harness around the UNMODIFIED reference estimator: CntHashEstimator from kmc_core/libs/ntHash/ntHashWrapper.h where it lies in the
// reference tree (nothing is copied).  __graft_entry__.build() compiles it into oracle/_ref/libkmc_nthash_ref.so; tests/estimate_testlib.py
// binds it.  It exists for s = 11, which the reference CLI takes only for inputs of at least 5 * 10^10 bytes.
//
// <math.h> comes first, as in the CLI's translation unit (kmc_runner.cpp): it brings std::abs(long) into the global namespace, so the
// estimator's abs((int64_t)...) is the 64-bit one there and here.
#include <math.h>
#include <cstdint>
#include <vector>
#include "kmc_core/libs/ntHash/ntHashWrapper.h"

// batch: kmcb200_split's format; every record (newline-separated) goes to Process on its own with A/C/G/T (either case) as 0..3 and every
// other byte as 255, as CSplitter::GetSeq codes it.  *n = max_occ + 1; out receives min(*n, cap) entries.
extern "C" int nthash_ref_histogram(const uint8_t* batch, uint64_t len, uint32_t k, uint32_t s, uint64_t* out, uint64_t cap, uint64_t* n)
{
	CntHashEstimator est(k, s);
	std::vector<char> codes;
	uint64_t start = 0;
	for (uint64_t i = 0; i <= len; ++i) {
		if (i < len && batch[i] != '\n') continue;
		codes.clear();
		for (uint64_t j = start; j < i; ++j) {
			const uint8_t c = batch[j];
			codes.push_back(c == 'A' || c == 'a' ? 0 : c == 'C' || c == 'c' ? 1 : c == 'G' || c == 'g' ? 2 : c == 'T' || c == 't' ? 3 : (char)-1);
		}
		if (!codes.empty()) est.Process(codes.data(), (uint32_t)codes.size());
		start = i + 1;
	}
	std::vector<uint64_t> hist;
	est.EstimateHistogram(hist);
	*n = hist.size();
	for (uint64_t i = 0; i < hist.size() && i < cap; ++i) out[i] = hist[i];
	return 0;
}
