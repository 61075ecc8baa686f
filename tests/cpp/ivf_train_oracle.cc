// TEST INFRASTRUCTURE.  FAISS's IVF training as reindexer::IvfIndex runs it (IvfIndex::trainIdx -> IndexIVFFlat::train(n, x, norms)),
// with the reference's vendored FAISS linked from oracle/_ref/liboracle_ref_ivf.so.  IndexIVFFlat::train normalises Cosine input and
// hands it to Level1Quantizer::train_q1, which runs a faiss::Clustering with the index's parameters on the quantizer and drops the
// Clustering; this oracle makes the same two calls itself so that the Clustering's iteration_stats survive.  Also rand_perm, the
// permutation the sample and the initial centroids come from.  Built by tests/cpp/ivf_train_oracle.mk where the reference tree exists;
// wrapped by tests/ivf_train_oracle.py.  The oracle's sgemm is a triple loop: keep shapes small.
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "faiss/Clustering.h"
#include "faiss/IndexFlat.h"
#include "faiss/IndexIVFFlat.h"
#include "faiss/utils/random.h"
#include "tools/normalize.h"

namespace {
thread_local std::string g_err;
}  // namespace

extern "C" {

const char* ivf_train_last_error() { return g_err.c_str(); }

void ivf_train_rand_perm(int32_t* perm, size_t n, int64_t seed) { faiss::rand_perm(perm, n, seed); }

// metric: 0 = L2, 1 = InnerProduct, 2 = Cosine (IvfIndex::newSpace / faissMetric).  norms: Cosine norm coefficients or NULL.
// out_centroids [nlist][dim]; obj / nsplit: one entry per iteration_stats entry, their number to *nstats (at most niter + 1)
int ivf_train_faiss(int metric, size_t dim, size_t nlist, size_t n, const float* vecs, const float* norms, int niter, int seed,
					int max_points_per_centroid, float* out_centroids, double* obj, int32_t* nsplit, int32_t* nstats) {
	try {
		std::unique_ptr<faiss::IndexFlat> space;
		if (metric == 0) {
			space = std::make_unique<faiss::IndexFlatL2>(dim);
		} else if (metric == 1) {
			space = std::make_unique<faiss::IndexFlatIP>(dim);
		} else if (metric == 2) {
			space = std::make_unique<faiss::IndexFlatCosine>(dim);
		} else {
			throw std::runtime_error("ivf_train_faiss: unknown metric");
		}
		faiss::IndexIVFFlat idx(space.get(), dim, nlist, metric == 0 ? faiss::METRIC_L2 : faiss::METRIC_INNER_PRODUCT, metric == 2);
		idx.cp.niter = niter;
		idx.cp.seed = seed;
		idx.cp.max_points_per_centroid = max_points_per_centroid;
		// IndexIVFFlat::train(n, x, x_norms): Cosine input times its norm coefficients, or normalised
		std::vector<float> x(vecs, vecs + n * dim);
		if (metric == 2) {
			for (size_t i = 0; i < n; ++i) {
				if (norms) {
					for (size_t j = 0; j < dim; ++j) {
						x[i * dim + j] *= norms[i];
					}
				} else {
					reindexer::ann::NormalizeVector(x.data() + i * dim, int32_t(dim));
				}
			}
		}
		// Level1Quantizer::train_q1, quantizer_trains_alone == 0
		faiss::Clustering clus(int(dim), int(nlist), idx.cp);
		space->reset();
		clus.train(faiss::idx_t(n), x.data(), *space);
		std::memcpy(out_centroids, clus.centroids.data(), nlist * dim * sizeof(float));
		*nstats = int32_t(clus.iteration_stats.size());
		for (size_t i = 0; i < clus.iteration_stats.size(); ++i) {
			obj[i] = clus.iteration_stats[i].obj;
			nsplit[i] = int32_t(clus.iteration_stats[i].nsplit);
		}
		return 0;
	} catch (const std::exception& e) {
		g_err = e.what();
	} catch (...) {
		g_err = "unknown exception";
	}
	return 1;
}

}  // extern "C"
