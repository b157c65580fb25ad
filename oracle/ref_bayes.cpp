// C wrapper over the reference's own rtabmap::BayesFilter (corelib/src/BayesFilter.cpp compiled against the stand-ins of
// oracle/refstubs/ into _ref/libref_bayes.so by `make ref`).  TEST INFRASTRUCTURE ONLY: the checker the GPU Bayes filter and
// oracle/bayes_py.py are compared against.
//
// The graph is the caller's: ref_bayes_set_graph loads, for every place, its neighbour table {id: margin} as
// Memory::getNeighborsId would return it, and the set of short-term-memory ids.
#include <cstdio>
#include <cstring>
#include <exception>
#include <map>
#include <string>
#include <vector>

#include "rtabmap/core/BayesFilter.h"
#include "rtabmap/core/Memory.h"

namespace {
struct RefBayes
{
	rtabmap::BayesFilter * bf = nullptr;
	rtabmap::Memory mem;
};
} // namespace

extern "C" {

// prediction_lc = NULL keeps the reference's default Bayes/PredictionLC
void * ref_bayes_create(const char * prediction_lc, float virtual_place_prior, int full_prediction_update)
{
	try
	{
		rtabmap::ParametersMap p;
		if (prediction_lc) p[rtabmap::Parameters::kBayesPredictionLC()] = prediction_lc;
		char vpp[32];
		std::snprintf(vpp, sizeof(vpp), "%.9g", static_cast<double>(virtual_place_prior)); // round-trips the float
		p[rtabmap::Parameters::kBayesVirtualPlacePriorThr()] = vpp;
		p[rtabmap::Parameters::kBayesFullPredictionUpdate()] = full_prediction_update ? "true" : "false";
		RefBayes * h = new RefBayes;
		h->bf = new rtabmap::BayesFilter(p);
		return h;
	}
	catch (const std::exception &)
	{
		return nullptr;
	}
}

void ref_bayes_destroy(void * h)
{
	RefBayes * r = static_cast<RefBayes *>(h);
	if (!r) return;
	delete r->bf;
	delete r;
}

// ids[n] places with a table; their neighbours are nbr_id/nbr_margin[ptr[i], ptr[i+1]); stm[n_stm] ids in the short-term memory
void ref_bayes_set_graph(void * h, const int * ids, int n, const long long * ptr, const int * nbr_id, const int * nbr_margin, const int * stm, int n_stm)
{
	RefBayes * r = static_cast<RefBayes *>(h);
	r->mem.neighbors.clear();
	r->mem.stm.clear();
	for (int i = 0; i < n; ++i)
	{
		std::map<int, int> & m = r->mem.neighbors[ids[i]];
		for (long long k = ptr[i]; k < ptr[i + 1]; ++k) m[nbr_id[k]] = nbr_margin[k];
	}
	for (int i = 0; i < n_stm; ++i) r->mem.stm.insert(stm[i]);
}

// BayesFilter::computePosterior; posterior_out[n] in id order.  Returns 0, or -1 when the reference threw (UFATAL / UASSERT).
int ref_bayes_compute_posterior(void * h, const int * ids, const float * likelihood, int n, float * posterior_out)
{
	RefBayes * r = static_cast<RefBayes *>(h);
	try
	{
		std::map<int, float> like;
		for (int i = 0; i < n; ++i) like[ids[i]] = likelihood[i];
		const std::map<int, float> & post = r->bf->computePosterior(&r->mem, like);
		int k = 0;
		for (const auto & kv : post)
			if (k < n) posterior_out[k++] = kv.second;
		return k == n ? 0 : -1;
	}
	catch (const std::exception &)
	{
		return -1;
	}
}

void ref_bayes_reset(void * h) { static_cast<RefBayes *>(h)->bf->reset(); }

// getPredictionLC: copies up to cap values, returns the pattern length
int ref_bayes_get_prediction_lc(void * h, double * out, int cap)
{
	const std::vector<double> & v = static_cast<RefBayes *>(h)->bf->getPredictionLC();
	for (int i = 0; i < cap && i < static_cast<int>(v.size()); ++i) out[i] = v[i];
	return static_cast<int>(v.size());
}

// BayesFilter::generatePrediction: the dense n x n float matrix, row-major (out[row * n + col]).  Returns 0, or -1 on a throw.
int ref_bayes_generate_prediction(void * h, const int * ids, int n, float * out)
{
	RefBayes * r = static_cast<RefBayes *>(h);
	try
	{
		const cv::Mat P = r->bf->generatePrediction(&r->mem, std::vector<int>(ids, ids + n));
		if (P.rows != n || P.cols != n) return -1;
		for (int row = 0; row < n; ++row) std::memcpy(out + static_cast<size_t>(row) * n, P.at_ptr(row, 0), n * sizeof(float));
		return 0;
	}
	catch (const std::exception &)
	{
		return -1;
	}
}

} // extern "C"
