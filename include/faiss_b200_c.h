/* faiss_b200 -- C ABI of the H100-native (sm_90a) similarity-search backend.
 *
 * Plain C (extern "C"), opaque handles, plain pointers and sizes; no torch / C++ types.
 * Two tiers:
 *   (1) index-level entry points with the names, argument meaning and error convention of the
 *       reference C API (c_api/Index_c.h:60-175, c_api/IndexShards_c.h:28-40,
 *       c_api/IndexIVF_c.h:118-160, c_api/gpu/StandardGpuResources_c.h, c_api/error_c.h:19-35):
 *       every function returns 0 on success, -2 for a Faiss-style exception (user error), -4 for a
 *       standard C++ exception, -1 otherwise; the message is read with faiss_get_last_error().
 *       The GPU index constructors, which the reference only exposes in C++
 *       (faiss/gpu/GpuIndexFlat.h:43-64, GpuIndexIVFFlat.h:37-59, GpuIndexIVFPQ.h:56-82), are
 *       exported here as faiss_GpuIndex*_new.
 *   (2) kernel-level seams (b200_*): device pointers + the resources' ordering stream, mirroring
 *       the reference's internal run* launchers (SURVEY.md section 8(b)).
 *
 * Pointer residency: for tier (1) every x / distances / labels / ids pointer may be host or
 * device memory (faiss/gpu/GpuIndex.cu:373-448).  Tier (2) takes DEVICE pointers only.
 * idx_t is int64_t (faiss/MetricType.h:52).
 */
#ifndef FAISS_B200_C_H
#define FAISS_B200_C_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define FB200_API __attribute__((visibility("default")))
#else
#define FB200_API
#endif

typedef int64_t idx_t;

typedef enum FaissErrorCode { /* c_api/error_c.h:19-30 */
    OK = 0,
    UNKNOWN_EXCEPT = -1,
    FAISS_EXCEPT = -2,
    STD_EXCEPT = -4
} FaissErrorCode;

typedef enum FaissMetricType { /* c_api/Index_c.h:26-36, faiss/MetricType.h:29-49 */
    METRIC_INNER_PRODUCT = 0,
    METRIC_L2 = 1,
    METRIC_L1 = 2,              /* GpuIndexFlat and bfKnn only, as the values below */
    METRIC_Linf = 3,
    METRIC_Lp = 4,              /* sum |a-b|^p with p = metric_arg (no root) */
    METRIC_Canberra = 20,
    METRIC_BrayCurtis = 21,
    METRIC_JensenShannon = 22,
    METRIC_Jaccard = 23,        /* a similarity: larger is better */
    METRIC_NaNEuclidean = 24,   /* declared, not implemented: "unimplemented metric type 24" */
    METRIC_GOWER = 25
} FaissMetricType;

typedef struct FaissIndex_H FaissIndex;                               /* c_api/Index_c.h:49 */
typedef struct FaissIndex_H FaissGpuIndex;
typedef struct FaissIndex_H FaissIndexShards;
typedef struct FaissStandardGpuResources_H FaissStandardGpuResources; /* c_api/gpu/StandardGpuResources_c.h:24 */

FB200_API const char* faiss_get_last_error(void);                    /* c_api/error_c.h:33 */
FB200_API const char* faiss_b200_version(void);

/* ---- StandardGpuResources (c_api/gpu/StandardGpuResources_c.h:24-55) ---- */
FB200_API int faiss_StandardGpuResources_new(FaissStandardGpuResources** p_res);
FB200_API void faiss_StandardGpuResources_free(FaissStandardGpuResources* res);
FB200_API int faiss_StandardGpuResources_noTempMemory(FaissStandardGpuResources* res);
FB200_API int faiss_StandardGpuResources_setTempMemory(FaissStandardGpuResources* res, size_t size);
FB200_API int faiss_StandardGpuResources_setPinnedMemory(FaissStandardGpuResources* res, size_t size);
FB200_API int faiss_StandardGpuResources_setDefaultStream(FaissStandardGpuResources* res, int device, void* cuda_stream);
FB200_API int faiss_StandardGpuResources_setDefaultNullStreamAllDevices(FaissStandardGpuResources* res);
/* c_api/gpu/GpuResources_c.h: getDefaultStream / syncDefaultStream */
FB200_API int faiss_StandardGpuResources_getDefaultStream(FaissStandardGpuResources* res, int device, void** out_stream);
FB200_API int faiss_StandardGpuResources_syncDefaultStream(FaissStandardGpuResources* res, int device);
/* getMemoryInfo (faiss/gpu/StandardGpuResources.h:243): writes a JSON object {dev:{type:[count,bytes]}} */
FB200_API int faiss_StandardGpuResources_getMemoryInfo(FaissStandardGpuResources* res, char* buf, size_t buflen);
FB200_API int faiss_StandardGpuResources_getTempMemoryAvailable(FaissStandardGpuResources* res, int device, size_t* out);

/* ---- generic Index (c_api/Index_c.h:49-175) ---- */
FB200_API void faiss_Index_free(FaissIndex* index);
FB200_API int faiss_Index_d(const FaissIndex* index);
FB200_API int faiss_Index_is_trained(const FaissIndex* index);
FB200_API idx_t faiss_Index_ntotal(const FaissIndex* index);
FB200_API FaissMetricType faiss_Index_metric_type(const FaissIndex* index);
/* faiss::Index::metric_arg (the exponent of METRIC_Lp); read at search time, so it may be set after add */
FB200_API float faiss_Index_metric_arg(const FaissIndex* index);
FB200_API void faiss_Index_set_metric_arg(FaissIndex* index, float metric_arg);
FB200_API int faiss_Index_verbose(const FaissIndex* index);
FB200_API void faiss_Index_set_verbose(FaissIndex* index, int v);
FB200_API int faiss_Index_train(FaissIndex* index, idx_t n, const float* x);
FB200_API int faiss_Index_add(FaissIndex* index, idx_t n, const float* x);
FB200_API int faiss_Index_add_with_ids(FaissIndex* index, idx_t n, const float* x, const idx_t* xids);
FB200_API int faiss_Index_search(const FaissIndex* index, idx_t n, const float* x, idx_t k, float* distances, idx_t* labels);
FB200_API int faiss_Index_assign(FaissIndex* index, idx_t n, const float* x, idx_t* labels, idx_t k);
FB200_API int faiss_Index_reset(FaissIndex* index);
FB200_API int faiss_Index_reconstruct(const FaissIndex* index, idx_t key, float* recons);
FB200_API int faiss_Index_reconstruct_n(const FaissIndex* index, idx_t i0, idx_t ni, float* recons);
FB200_API int faiss_Index_reconstruct_batch(const FaissIndex* index, idx_t n, const idx_t* keys, float* recons);
FB200_API int faiss_Index_compute_residual(const FaissIndex* index, const float* x, float* residual, idx_t key);
FB200_API int faiss_Index_compute_residual_n(const FaissIndex* index, idx_t n, const float* x, float* residuals, const idx_t* keys);

/* GpuIndex::setMinPagingSize / getMinPagingSize (faiss/gpu/GpuIndex.h:66-69): host-resident query blocks of at least
 * this many bytes (default 256 MiB) are paged through the resources' pinned buffer, H2D of page p+1 overlapping the
 * search of page p (role of searchFromCpuPaged_, faiss/gpu/GpuIndex.cu:620-788). */
FB200_API int faiss_GpuIndex_setMinPagingSize(FaissGpuIndex* index, size_t size);
FB200_API int faiss_GpuIndex_getMinPagingSize(const FaissGpuIndex* index, size_t* out_size);

/* ---- GpuIndexFlat (faiss/gpu/GpuIndexFlat.h:43-217) ---- */
/* use_tensor_cores: 1 = tensor-core path when the shape supports it (default), 0 = exact SIMT only */
FB200_API int faiss_GpuIndexFlat_new(FaissGpuIndex** p_index, FaissStandardGpuResources* res, int d, FaissMetricType metric, int device, int use_tensor_cores);
/* GpuIndexFlatConfig (faiss/gpu/GpuIndexFlat.h:26-35).  use_float16: the vectors are stored as fp16 and queries are
 * rounded to fp16 before the comparison, as FlatIndex::query does (faiss/gpu/impl/FlatIndex.cu:112-136); distances are
 * the exact fp32 distances between the rounded values. */
FB200_API int faiss_GpuIndexFlat_new_with_config(FaissGpuIndex** p_index, FaissStandardGpuResources* res, int d, FaissMetricType metric, int device, int use_tensor_cores, int use_float16);
FB200_API int faiss_GpuIndexFlatL2_new(FaissGpuIndex** p_index, FaissStandardGpuResources* res, int d, int device);
FB200_API int faiss_GpuIndexFlatIP_new(FaissGpuIndex** p_index, FaissStandardGpuResources* res, int d, int device);
/* copyFrom / copyTo against the CPU IndexFlat payload (faiss/gpu/GpuIndexFlat.cu:105-176) */
FB200_API int faiss_GpuIndexFlat_copyFrom(FaissGpuIndex* index, idx_t n, const float* xb);
FB200_API int faiss_GpuIndexFlat_copyTo(const FaissGpuIndex* index, float* xb_out);
FB200_API int faiss_GpuIndexFlat_setUseTensorCores(FaissGpuIndex* index, int enable);
/* diagnostics of the last search on this index: out[0] = tensor-core path used, out[1] = queries
   recomputed by the exact kernel because their certificate failed */
FB200_API int faiss_GpuIndexFlat_lastSearchInfo(const FaissGpuIndex* index, int* out2);
/* operand width of the last search's tensor-core scoring: 8 (int8), 16 (fp16), or 0 when it ran the exact kernel */
FB200_API int faiss_GpuIndexFlat_lastSearchOperandBits(const FaissGpuIndex* index, int* bits);

/* ---- GpuIndexIVF (faiss/gpu/GpuIndexIVF.h:40-167) ---- */
FB200_API int faiss_GpuIndexIVF_set_nprobe(FaissGpuIndex* index, size_t nprobe);
FB200_API size_t faiss_GpuIndexIVF_nprobe(const FaissGpuIndex* index);
FB200_API size_t faiss_GpuIndexIVF_nlist(const FaissGpuIndex* index);
FB200_API int faiss_GpuIndexIVF_set_clustering(FaissGpuIndex* index, int niter, int seed, int max_points_per_centroid);
FB200_API int faiss_GpuIndexIVF_reserveMemory(FaissGpuIndex* index, size_t num_vecs);
FB200_API int faiss_GpuIndexIVF_reclaimMemory(FaissGpuIndex* index, size_t* reclaimed);
FB200_API size_t faiss_GpuIndexIVF_get_list_size(const FaissGpuIndex* index, size_t list_no); /* c_api/IndexIVF_c.h:129 */
/* getListVectorData / getListIndices (faiss/gpu/GpuIndexIVF.h:120-130): host output buffers */
FB200_API int faiss_GpuIndexIVF_getListVectorData(const FaissGpuIndex* index, size_t list_no, uint8_t* codes_out);
FB200_API int faiss_GpuIndexIVF_getListIndices(const FaissGpuIndex* index, size_t list_no, idx_t* ids_out);
/* copyFrom pieces (faiss/gpu/GpuIndexIVF.cu copyFrom, IVFBase.cu:328-451): coarse centroids and
   ArrayInvertedLists-format lists */
FB200_API int faiss_GpuIndexIVF_setCoarseCentroids(FaissGpuIndex* index, const float* centroids);
FB200_API int faiss_GpuIndexIVF_getCoarseCentroids(const FaissGpuIndex* index, float* centroids_out);
FB200_API int faiss_GpuIndexIVF_setList(FaissGpuIndex* index, size_t list_no, idx_t len, const uint8_t* codes, const idx_t* ids);
/* bulk clone: exact capacity for all nlist lists in ONE arena relayout, to be called before the nlist
   setList calls (lens: host, [nlist]) -- the per-list reserve of IVFBase::copyInvertedListsFrom
   (faiss/gpu/impl/IVFBase.cu:328-451) */
FB200_API int faiss_GpuIndexIVF_setListSizes(FaissGpuIndex* index, const idx_t* lens);
FB200_API int faiss_GpuIndexIVF_set_is_trained(FaissGpuIndex* index, int v);
/* c_api/IndexIVF_c.h:118 faiss_IndexIVF_search_preassigned */
FB200_API int faiss_GpuIndexIVF_search_preassigned(const FaissGpuIndex* index, idx_t n, const float* x, idx_t k, const idx_t* assign, const float* centroid_dis, float* distances, idx_t* labels);

FB200_API int faiss_GpuIndexIVFFlat_new(FaissGpuIndex** p_index, FaissStandardGpuResources* res, int d, idx_t nlist, FaissMetricType metric, int device);

/* ---- GpuIndexIVFPQ (faiss/gpu/GpuIndexIVFPQ.h:56-181) ---- */
FB200_API int faiss_GpuIndexIVFPQ_new(FaissGpuIndex** p_index, FaissStandardGpuResources* res, int d, idx_t nlist, idx_t M, idx_t nbits, FaissMetricType metric, int device);
/* GpuIndexIVFPQConfig::interleavedLayout (faiss/gpu/GpuIndexIVFPQ.h:36-40): with interleaved_layout != 0, nbits
   may be 4, 5, 6 or 8 (else only 8); lists hold ceil(M * nbits / 8) code bytes per vector, the CPU's packed
   bitstring.  coarse: a GpuIndexFlat to share as the coarse quantizer, or NULL. */
FB200_API int faiss_GpuIndexIVFPQ_new_with_config(FaissGpuIndex** p_index, FaissStandardGpuResources* res, FaissGpuIndex* coarse /* nullable */, int d, idx_t nlist, idx_t M, idx_t nbits, FaissMetricType metric, int device, int interleaved_layout);
FB200_API int faiss_GpuIndexIVFPQ_setPQCentroids(FaissGpuIndex* index, const float* centroids /* [M][2^nbits][dsub] */);
FB200_API int faiss_GpuIndexIVFPQ_getPQCentroids(const FaissGpuIndex* index, float* centroids_out /* [M][2^nbits][dsub] */);
FB200_API int faiss_GpuIndexIVFPQ_set_pq_clustering(FaissGpuIndex* index, int niter, int seed, int max_points_per_centroid);
/* GpuIndexIVFPQ::setPrecomputedCodes (faiss/gpu/GpuIndexIVFPQ.h:114-118): force the precomputed term-2 table
   ([nlist][256][M] floats, L2 only) on or off; untouched, the index follows the CPU reference's "auto" size
   rule (<= 2 GiB, faiss/IndexIVFPQ.cpp:345) for indexes with short lists.  Results agree to fp32 rounding. */
FB200_API int faiss_GpuIndexIVFPQ_setPrecomputedCodes(FaissGpuIndex* index, int enable);

/* ---- GpuIndexIVFScalarQuantizer (faiss/gpu/GpuIndexIVFScalarQuantizer.h:30-139) ----
   qtype: ScalarQuantizer::QuantizerType 0-6 (QT_8bit, QT_4bit, QT_8bit_uniform, QT_4bit_uniform, QT_fp16,
   QT_8bit_direct, QT_6bit); any other type fails with "Unsupported scalar QuantizerType on GPU".
   trained: ScalarQuantizer::trained ([vmin, vdiff] uniform, [vmin[d], vdiff[d]] non-uniform, empty for fp16 and
   8bit_direct).  get_trained writes *n values to out when out is non-NULL; pass NULL to query the length.
   Lists, nprobe, reserve and search go through faiss_GpuIndexIVF_* and faiss_Index_*. */
FB200_API int faiss_GpuIndexIVFScalarQuantizer_new(FaissGpuIndex** p_index, FaissStandardGpuResources* res, int d, idx_t nlist, int qtype, FaissMetricType metric, int encodeResidual, int device);
FB200_API int faiss_GpuIndexIVFScalarQuantizer_new_with_quantizer(FaissGpuIndex** p_index, FaissStandardGpuResources* res, FaissGpuIndex* coarse, int d, idx_t nlist, int qtype, FaissMetricType metric, int encodeResidual, int device);
FB200_API int faiss_GpuIndexIVFScalarQuantizer_set_trained(FaissGpuIndex* index, const float* trained, size_t n);
FB200_API int faiss_GpuIndexIVFScalarQuantizer_get_trained(const FaissGpuIndex* index, float* out, size_t* n);
FB200_API int faiss_GpuIndexIVFScalarQuantizer_code_size(const FaissGpuIndex* index, size_t* out);
FB200_API int faiss_GpuIndexIVFScalarQuantizer_qtype(const FaissGpuIndex* index, int* out);
FB200_API int faiss_GpuIndexIVFScalarQuantizer_by_residual(const FaissGpuIndex* index, int* out);
/* ScalarQuantizer::rangestat / rangestat_arg used by train(); only RS_minmax (0) trains on the GPU */
FB200_API int faiss_GpuIndexIVFScalarQuantizer_set_rangestat(FaissGpuIndex* index, int rangestat, float rangestat_arg);

/* ---- IndexShards (c_api/IndexShards_c.h:28-40) ---- */
FB200_API int faiss_IndexShards_new(FaissIndexShards** p_index, idx_t d);
FB200_API int faiss_IndexShards_new_with_options(FaissIndexShards** p_index, idx_t d, int threaded, int successive_ids);
FB200_API int faiss_IndexShards_add_shard(FaissIndexShards* index, FaissIndex* shard);
FB200_API int faiss_IndexShards_remove_shard(FaissIndexShards* index, FaissIndex* shard);
FB200_API FaissIndex* faiss_IndexShards_at(FaissIndexShards* index, int i);
FB200_API int faiss_IndexShards_own_indices(const FaissIndexShards* index);
FB200_API void faiss_IndexShards_set_own_indices(FaissIndexShards* index, int v);
FB200_API int faiss_IndexShards_successive_ids(const FaissIndexShards* index);
FB200_API void faiss_IndexShards_set_successive_ids(FaissIndexShards* index, int v);

/* ---- SearchParameters (faiss/Index.h:88-93, faiss/IndexIVF.h:68-90; c_api/IndexIVF_c.h faiss_SearchParametersIVF_new_with),
   InterruptCallback (faiss/impl/AuxIndexStructures.h), constructors sharing a coarse quantiser
   (faiss/gpu/GpuIndexIVFFlat.h:48-59, GpuIndexIVFPQ.h:69-82) ---- */
typedef struct FaissSearchParameters_H FaissSearchParameters;
typedef struct FaissSearchParameters_H FaissSearchParametersIVF;
FB200_API int faiss_SearchParametersIVF_new_with(FaissSearchParametersIVF** p_sp, size_t nprobe, size_t max_codes);
FB200_API void faiss_SearchParameters_free(FaissSearchParameters* sp);

/* ---- IDSelector (c_api/impl/AuxIndexStructures_c.h names and argument order; faiss/impl/IDSelector.h semantics).
   A selector restricts a search to the stored ids it accepts: the row number for GpuIndexFlat, the id stored
   in the list (add_with_ids) for the IVF indexes, whose coarse search is not filtered.  Leaves copy their
   inputs; Not / And / Or / XOr keep pointers to their operands, which must outlive them.  Array and Batch
   select by membership (duplicates and ids past ntotal are harmless); an empty Range selects nothing. ---- */
typedef struct FaissIDSelector_H FaissIDSelector;
typedef struct FaissIDSelector_H FaissIDSelectorRange;
typedef struct FaissIDSelector_H FaissIDSelectorArray;
typedef struct FaissIDSelector_H FaissIDSelectorBatch;
typedef struct FaissIDSelector_H FaissIDSelectorBitmap;
typedef struct FaissIDSelector_H FaissIDSelectorNot;
typedef struct FaissIDSelector_H FaissIDSelectorAnd;
typedef struct FaissIDSelector_H FaissIDSelectorOr;
typedef struct FaissIDSelector_H FaissIDSelectorXOr;
FB200_API void faiss_IDSelector_free(FaissIDSelector* sel);
/* 1 if id is selected, 0 if not, -1 on a null handle */
FB200_API int faiss_IDSelector_is_member(const FaissIDSelector* sel, idx_t id);
FB200_API int faiss_IDSelectorRange_new(FaissIDSelectorRange** p_sel, idx_t imin, idx_t imax);
FB200_API int faiss_IDSelectorArray_new(FaissIDSelectorArray** p_sel, size_t n, const idx_t* ids);
FB200_API int faiss_IDSelectorBatch_new(FaissIDSelectorBatch** p_sel, size_t n, const idx_t* indices);
/* bit (id & 7) of byte id >> 3, for id >> 3 < n */
FB200_API int faiss_IDSelectorBitmap_new(FaissIDSelectorBitmap** p_sel, size_t n, const uint8_t* bitmap);
FB200_API int faiss_IDSelectorNot_new(FaissIDSelectorNot** p_sel, const FaissIDSelector* sel);
FB200_API int faiss_IDSelectorAnd_new(FaissIDSelectorAnd** p_sel, const FaissIDSelector* lhs_sel, const FaissIDSelector* rhs_sel);
FB200_API int faiss_IDSelectorOr_new(FaissIDSelectorOr** p_sel, const FaissIDSelector* lhs_sel, const FaissIDSelector* rhs_sel);
FB200_API int faiss_IDSelectorXOr_new(FaissIDSelectorXOr** p_sel, const FaissIDSelector* lhs_sel, const FaissIDSelector* rhs_sel);
/* a selector this library cannot see into: is_member(id) = (is_member(ctx, id) != 0), called on the host once per
   stored entry and search call */
FB200_API int faiss_b200_IDSelectorCallback_new(FaissIDSelector** p_sel, int (*is_member)(void* ctx, idx_t id), void* ctx);
/* c_api/Index_c.h:44 and c_api/IndexIVF_c.h faiss_SearchParametersIVF_new_with: sel may be NULL and is not owned */
FB200_API int faiss_SearchParameters_new(FaissSearchParameters** p_sp, FaissIDSelector* sel);
FB200_API int faiss_SearchParametersIVF_new_with_sel(FaissSearchParametersIVF** p_sp, FaissIDSelector* sel, size_t nprobe, size_t max_codes);

/* ---- GpuIndexCagra (faiss/gpu/GpuIndexCagra.h:41-380): fp32, METRIC_L2 / METRIC_INNER_PRODUCT, one GPU.
   The configuration structs flatten GpuIndexCagraConfig with its IVFPQBuildCagraConfig / IVFPQSearchCagraConfig
   and SearchParametersCagra; enums take the reference's values (graph_build_algo IVF_PQ = 0, NN_DESCENT = 1,
   ITERATIVE_SEARCH = 2; codebook_gen PER_SUBSPACE = 0, PER_CLUSTER = 1; search_algo SINGLE_CTA = 0, MULTI_CTA = 1,
   MULTI_KERNEL = 2, AUTO = 100; hash_mode HASH = 0, SMALL = 1, AUTO = 100).  Search goes through
   faiss_Index_search_with_params with a FaissSearchParametersCagra (or faiss_Index_search: the defaults). ---- */
typedef struct FaissGpuIndexCagraConfig {
    int device;
    size_t intermediate_graph_degree; /* 128 */
    size_t graph_degree;              /* 64 */
    int build_algo;                   /* 0 */
    size_t nn_descent_niter;          /* 20 */
    float refine_rate;                /* 2.0 */
    int store_dataset;                /* 1 */
    int guarantee_connectivity;       /* 0 */
    /* IVFPQBuildCagraConfig */
    uint32_t n_lists;                 /* 1024 */
    uint32_t kmeans_n_iters;          /* 20 */
    double kmeans_trainset_fraction;  /* 0.5 */
    uint32_t pq_bits;                 /* 8 */
    uint32_t pq_dim;                  /* 0 */
    int codebook_kind;                /* 0 */
    int force_random_rotation;        /* 0 */
    int conservative_memory_allocation; /* 0 */
    /* IVFPQSearchCagraConfig */
    uint32_t n_probes;                /* 20 */
    uint32_t max_internal_batch_size; /* 4096 */
} FaissGpuIndexCagraConfig;
/* the reference's defaults */
FB200_API void faiss_GpuIndexCagraConfig_init(FaissGpuIndexCagraConfig* config);
FB200_API int faiss_GpuIndexCagra_new(FaissGpuIndex** p_index, FaissStandardGpuResources* res, int d, FaissMetricType metric, const FaissGpuIndexCagraConfig* config);
/* graph [ntotal][degree] as int64 (-1: no edge) */
FB200_API int faiss_GpuIndexCagra_graph_degree(const FaissGpuIndex* index, int* degree);
FB200_API int faiss_GpuIndexCagra_get_knngraph(const FaissGpuIndex* index, idx_t* graph);
/* the IndexHNSWCagra payload: xb [n][d], graph [n][degree] (level 0; -1 entries are skipped by the search) */
FB200_API int faiss_GpuIndexCagra_copyFrom(FaissGpuIndex* index, idx_t n, const float* xb, const idx_t* graph, int degree);
FB200_API int faiss_GpuIndexCagra_copyTo(const FaissGpuIndex* index, float* xb, idx_t* graph);
/* distance evaluations of the last search; seconds of the last build (IVF-PQ candidates, refine, optimise) */
FB200_API int faiss_GpuIndexCagra_lastSearchDistanceCount(const FaissGpuIndex* index, int64_t* count);
FB200_API int faiss_GpuIndexCagra_lastBuildSeconds(const FaissGpuIndex* index, double* seconds3);

typedef struct FaissSearchParametersCagraConfig {
    size_t max_queries;           /* 0 */
    size_t itopk_size;            /* 64 */
    size_t max_iterations;        /* 0 */
    int algo;                     /* 100 */
    size_t team_size;             /* 0 */
    size_t search_width;          /* 1 */
    size_t min_iterations;        /* 0 */
    size_t thread_block_size;     /* 0 */
    int hashmap_mode;             /* 100 */
    size_t hashmap_min_bitlen;    /* 0 */
    float hashmap_max_fill_rate;  /* 0.5 */
    uint32_t num_random_samplings; /* 1 */
    uint64_t seed;                /* 0x128394 */
} FaissSearchParametersCagraConfig;
typedef struct FaissSearchParameters_H FaissSearchParametersCagra;
FB200_API void faiss_SearchParametersCagraConfig_init(FaissSearchParametersCagraConfig* config);
/* sel may be NULL (GpuIndexCagra rejects a selector at search time) */
FB200_API int faiss_SearchParametersCagra_new(FaissSearchParametersCagra** p_sp, FaissIDSelector* sel, const FaissSearchParametersCagraConfig* config);

/* the graph optimisation of the GpuIndexCagra build on its own (device pointers, uint32 ids): G0 [n][K0] -> G [n][K].
   Every G0 row must hold K0 distinct ids other than its own row; 1 <= K <= K0 <= 1024.  An entry >= n (such as a -1)
   or equal to its own row is an error, reported before G is written. */
FB200_API int b200_cagra_optimize(FaissStandardGpuResources* res, int device, const uint32_t* G0, int64_t n, int K0, int K, uint32_t* G);

/* c_api/Index_c.h faiss_Index_search_with_params: per-call nprobe for IVF indexes (max_codes must be 0) and an
   IDSelector for GPU indexes */
FB200_API int faiss_Index_search_with_params(const FaissIndex* index, idx_t n, const float* x, idx_t k, const FaissSearchParameters* params, float* distances, idx_t* labels);
/* faiss::Index::search_and_reconstruct (GpuIndexFlat and the IVF indexes; params may be NULL): distances / labels as
   faiss_Index_search_with_params, recons [n][k][d] the stored vector of each result (all 0xFF bytes for label -1).
   IVF: the entry the search returned, decoded as IndexIVF::reconstruct_from_offset. */
FB200_API int faiss_Index_search_and_reconstruct(const FaissIndex* index, idx_t n, const float* x, idx_t k, const FaissSearchParameters* params, float* distances, idx_t* labels, float* recons);
/* faiss::IndexIVF::search_and_return_codes: codes [n][k][(include_listno ? coarse code size : 0) + code size], the
   CPU inverted-list bytes of each result, prefixed by its list number (little-endian); all 0xFF for label -1 */
FB200_API int faiss_GpuIndexIVF_search_and_return_codes(const FaissGpuIndex* index, idx_t n, const float* x, idx_t k, const FaissSearchParameters* params, float* distances, idx_t* labels, uint8_t* codes, int include_listno);
/* IndexIVF::coarse_code_size and code_size: the byte widths of a search_and_return_codes row */
FB200_API int faiss_GpuIndexIVF_code_sizes(const FaissGpuIndex* index, int* coarse_code_size, int* code_size);
/* polled between query pages, add pages and clustering iterations; non-zero return -> the running call fails with
   "computation interrupted" (-2).  NULL clears it. */
FB200_API void faiss_b200_set_interrupt_callback(int (*want_interrupt)(void* ctx), void* ctx);
/* `coarse` = a GpuIndexFlat of this library on the same device (shared, not owned); the index is trained iff it
   already holds nlist centroids (an IVFPQ still needs train() for its PQ) */
FB200_API int faiss_GpuIndexIVFFlat_new_with_quantizer(FaissGpuIndex** p_index, FaissStandardGpuResources* res, FaissGpuIndex* coarse, int d, idx_t nlist, FaissMetricType metric, int device);
FB200_API int faiss_GpuIndexIVFPQ_new_with_quantizer(FaissGpuIndex** p_index, FaissStandardGpuResources* res, FaissGpuIndex* coarse, int d, idx_t nlist, idx_t M, idx_t nbits, FaissMetricType metric, int device);

/* ---- NCCL communicator ownership + IndexShards across ranks ----
   The reference shards over the GPUs of a box with IndexShards (one worker thread per sub-index, host heap
   merge: faiss/IndexShards.cpp:197-264, faiss/impl/ThreadedIndex-inl.h:119-194); ToGpuClonerMultiple builds it
   (faiss/gpu/GpuCloner.cpp:418-436).  Here the resources object owns one NCCL communicator per device:
     ncclInitAll  -- all listed devices of THIS process form one clique (rank i = devices[i]); an IndexShards
                     whose shards are GpuIndexes on exactly those devices, in rank order, then searches with
                     per-device threads + one ncclAllGather + a device merge instead of the host merge;
     ncclInitRank -- this process is rank `rank` of `nranks` (one process per GPU); the 128-byte id comes from
                     faiss_b200_nccl_unique_id on one rank and reaches the others through the launcher.
   faiss_DistributedIndexShards = IndexShards with ONE shard per rank: faiss_Index_search on it is a
   collective call (identical queries and k on every rank), results on every rank; add() adds to the local
   shard.  b200_shards_search is the one-shot kernel-seam form (SURVEY 8(b)). */
FB200_API int faiss_b200_nccl_unique_id(char* out128);
FB200_API int faiss_StandardGpuResources_ncclInitRank(FaissStandardGpuResources* res, int device, int nranks, int rank, const char* unique_id128);
FB200_API int faiss_StandardGpuResources_ncclInitAll(FaissStandardGpuResources* res, int ndev, const int* devices);
FB200_API int faiss_StandardGpuResources_ncclRank(FaissStandardGpuResources* res, int device, int* rank, int* nranks);
/* faiss::IndexShardsIVF (faiss/IndexShardsIVF.cpp:100-251; GpuMultipleClonerOptions::common_ivf_quantizer,
   faiss/gpu/GpuCloner.cpp:418-436): IVF shards over ONE shared coarse quantiser -- the coarse search runs once, every
   shard scans through search_preassigned, results are merged.  `quantizer` = a GpuIndexFlat (shared, not owned). */
FB200_API int faiss_IndexShardsIVF_new(FaissIndexShards** p_index, FaissGpuIndex* quantizer, idx_t nlist, int threaded, int successive_ids);
FB200_API int faiss_IndexShardsIVF_add_shard(FaissIndexShards* index, FaissIndex* shard);
/* path of the last faiss_Index_search on an IndexShards: 0 = thread per shard + host merge, 1 = NCCL fast path */
FB200_API int faiss_IndexShards_lastSearchPath(const FaissIndexShards* index);
FB200_API int faiss_DistributedIndexShards_new(FaissIndexShards** p_index, FaissStandardGpuResources* res, FaissGpuIndex* local_shard, int successive_ids);
FB200_API int faiss_DistributedIndexShards_sync(FaissIndexShards* index); /* collective: re-read every shard's ntotal */
FB200_API int faiss_DistributedIndexShards_info(const FaissIndexShards* index, int* rank, int* nranks, idx_t* id_offset);
FB200_API int b200_shards_search(FaissStandardGpuResources* res, FaissGpuIndex* local_shard, int successive_ids, idx_t n, const float* x, idx_t k, float* distances, idx_t* labels);

/* ---- GpuIcmEncoder (faiss/gpu/GpuIcmEncoder.h; faiss/impl/LocalSearchQuantizer.cpp:539-795) ----
   LocalSearchQuantizer's ICM encoding (lsq::IcmEncoder::encode) on one or more devices, rows split into contiguous
   ranges.  The perturbation draws are the caller's: perturbations is [ils_iters][n][nperts] pairs (m, k) as int32,
   drawn in the order of LocalSearchQuantizer::perturb_codes, so a caller that draws them from its std::mt19937 follows
   the CPU encoder's random trajectory.  codes [n][M] int32 (in: start codes, out: best codes), x [n][d] and
   perturbations may each be host or device memory.  Limits: 1 <= K <= 1024, nperts <= M. */
typedef struct FaissGpuIcmEncoder_H FaissGpuIcmEncoder;
/* res[i] serves devices[i]; each device needs a resources object of its own */
FB200_API int faiss_GpuIcmEncoder_new(FaissGpuIcmEncoder** p_enc, int M, int K, int d, int ndevices, FaissStandardGpuResources** res, const int* devices);
FB200_API void faiss_GpuIcmEncoder_free(FaissGpuIcmEncoder* enc);
/* codebooks [M][K][d] (host or device): lsq::IcmEncoder::set_binary_term */
FB200_API int faiss_GpuIcmEncoder_set_binary_term(FaissGpuIcmEncoder* enc, const float* codebooks);
FB200_API int faiss_GpuIcmEncoder_encode(FaissGpuIcmEncoder* enc, int32_t* codes, const float* x, idx_t n, size_t ils_iters, size_t nperts, size_t icm_iters, const int32_t* perturbations);
/* faiss_GpuIcmEncoder_encode with a page budget of page_bytes instead of 256 MiB */
FB200_API int b200_icm_encode_paged(FaissGpuIcmEncoder* enc, int32_t* codes, const float* x, idx_t n, size_t ils_iters, size_t nperts, size_t icm_iters, const int32_t* perturbations, size_t page_bytes);

/* ---- GpuRqEncoder (faiss/impl/ResidualQuantizer.cpp:432-520; faiss/impl/residual_quantizer_encode_steps.cpp) ----
   ResidualQuantizer's beam-search encoding on one device, in both distance modes.  nbits[m] in [1, 12]; every beam in
   [1, 256].  Every pointer may be host or device memory.  B below is the beam after the M steps,
   min(beam_in * prod 2^nbits, out_beam) (faiss_b200_RqEncoder_final_beam). */
typedef struct FaissGpuRqEncoder_H FaissGpuRqEncoder;
FB200_API int faiss_b200_RqEncoder_new(FaissGpuRqEncoder** p_enc, FaissStandardGpuResources* res, int device, int d, int M, const int* nbits);
FB200_API void faiss_b200_RqEncoder_free(FaissGpuRqEncoder* enc);
/* codebooks [total_K][d]: the device copy, the centroid norms and the per-step cross-product blocks */
FB200_API int faiss_b200_RqEncoder_set_codebooks(FaissGpuRqEncoder* enc, const float* codebooks);
FB200_API int faiss_b200_RqEncoder_final_beam(const FaissGpuRqEncoder* enc, int beam_in, int out_beam, int* beam);
/* ResidualQuantizer::refine_beam (use_beam_LUT = 0): residuals [n][beam_in][d] -> codes [n][B][M], residuals_out
   [n][B][d], distances [n][B]; each output may be NULL */
FB200_API int faiss_b200_RqEncoder_refine_beam(FaissGpuRqEncoder* enc, idx_t n, int beam_in, const float* residuals, int out_beam, int32_t* codes, float* residuals_out, float* distances);
/* ResidualQuantizer::refine_beam_LUT (use_beam_LUT = 1), given x [n][d] instead of (query_norms, query_cp): the device
   computes both.  codes [n][B][M], distances [n][B]; each may be NULL */
FB200_API int faiss_b200_RqEncoder_refine_beam_lut(FaissGpuRqEncoder* enc, idx_t n, const float* x, int out_beam, int32_t* codes, float* distances);
/* ResidualQuantizer::compute_codes_add_centroids with out_beam_size max_beam: packed [n][code_size] for search_type
   ST_decompress, ST_LUT_nonorm, ST_norm_from_LUT, ST_norm_float, ST_norm_qint8 or ST_norm_qint4 (0 .. 5); the other
   search types return an error.  centroids [n][d] or NULL. */
FB200_API int faiss_b200_RqEncoder_compute_codes(FaissGpuRqEncoder* enc, const float* x, idx_t n, int use_beam_lut, int max_beam, int search_type, float norm_min, float norm_max, const float* centroids, uint8_t* packed);
/* the same search, unpacked: codes [n][M] (entry 0 of the beam), for a caller that packs with a search type the
   device does not */
FB200_API int faiss_b200_RqEncoder_encode_unpacked(FaissGpuRqEncoder* enc, const float* x, idx_t n, int use_beam_lut, int max_beam, int32_t* codes);
/* refine_beam, refine_beam_lut and compute_codes with a page budget of page_bytes instead of 256 MiB */
FB200_API int b200_rq_refine_beam_paged(FaissGpuRqEncoder* enc, idx_t n, int beam_in, const float* residuals, int out_beam, int32_t* codes, float* residuals_out, float* distances, size_t page_bytes);
FB200_API int b200_rq_refine_beam_lut_paged(FaissGpuRqEncoder* enc, idx_t n, const float* x, int out_beam, int32_t* codes, float* distances, size_t page_bytes);
FB200_API int b200_rq_compute_codes_paged(FaissGpuRqEncoder* enc, const float* x, idx_t n, int use_beam_lut, int max_beam, int search_type, float norm_min, float norm_max, const float* centroids, uint8_t* packed, size_t page_bytes);

/* ---- Clustering (c_api/Clustering_c.h faiss_kmeans_clustering; faiss/Clustering.cpp:60-380) ----
   Lloyd k-means with the training set resident on the device; x host or device. */
FB200_API int faiss_b200_kmeans(FaissStandardGpuResources* res, int device, size_t d, size_t n, size_t k, const float* x, int niter, int seed, int max_points_per_centroid, float* centroids_out /* host [k*d] */, float* obj_out /* host [niter] or NULL */);

/* same with the assignment metric and ClusteringParameters::spherical (what GpuIndexIVF uses for
   METRIC_INNER_PRODUCT, faiss/gpu/GpuIndexIVF.cu:72-76; post_process_centroids, faiss/Clustering.cpp:35-45) */
FB200_API int faiss_b200_kmeans_ex(FaissStandardGpuResources* res, int device, size_t d, size_t n, size_t k, const float* x, int niter, int seed, int max_points_per_centroid, FaissMetricType metric, int spherical, float* centroids_out, float* obj_out);
/* Lloyd k-means with the training set sharded over the ranks of the device's NCCL communicator (collective call:
   every rank passes its own rows, rank order = row order of the concatenated set; faiss/Clustering.cpp:60-380 on the
   concatenation, SURVEY 8(e)): local Flat k=1 assignment, deterministic local partial sums, ONE packed ncclAllReduce
   per iteration (k*d sums | k counts | objective), identical split_clusters on every rank.  centroids_out host [k*d]
   (identical on all ranks); stats_out (optional, 4 doubles): total s, s in search+update+all-reduce, s in
   split_clusters, number of splits */
FB200_API int faiss_b200_kmeans_sharded(FaissStandardGpuResources* res, int device, size_t d, size_t n_local, size_t k, const float* x_local, int niter, int seed, float* centroids_out, float* obj_out, double* stats_out);
/* ProductQuantizer::train, Train_default (faiss/impl/ProductQuantizer.cpp:130-195): M independent 256-centroid
   k-means on the column slices of x [n,d] (host or device); centroids_out host [M][256][d/M] */
FB200_API int faiss_b200_pq_train(FaissStandardGpuResources* res, int device, size_t d, size_t M, size_t n, const float* x, int niter, int seed, float* centroids_out);

/* bfKnn (faiss/gpu/GpuDistance.h:33-181): brute-force k-NN of `queries` in `vectors` (both row-major fp32, host or
   device), any metric GpuIndexFlat takes; outputs host or device.  fp16 / bf16 and column-major inputs, int32 ids,
   all pairwise distances (k = -1) and tiling: faiss_b200_bfKnn_params / faiss_b200_bfKnn_tiling below. */
FB200_API int faiss_b200_bfKnn(FaissStandardGpuResources* res, int device, FaissMetricType metric, idx_t k, int dims, const float* vectors, idx_t num_vectors, const float* queries, idx_t num_queries, float* out_distances, idx_t* out_indices);
/* the same with GpuDistanceParams::metricArg (faiss/gpu/GpuDistance.h:41), the exponent of METRIC_Lp */
FB200_API int faiss_b200_bfKnn_ex(FaissStandardGpuResources* res, int device, FaissMetricType metric, float metric_arg, idx_t k, int dims, const float* vectors, idx_t num_vectors, const float* queries, idx_t num_queries, float* out_distances, idx_t* out_indices);

/* faiss::gpu::DistanceDataType / IndicesDataType (faiss/gpu/GpuDistance.h:18-29), same values */
typedef enum FaissDistanceDataType {
    FaissDistanceDataType_F32 = 1,
    FaissDistanceDataType_F16 = 2,
    FaissDistanceDataType_BF16 = 3
} FaissDistanceDataType;
typedef enum FaissIndicesDataType {
    FaissIndicesDataType_I64 = 1,
    FaissIndicesDataType_I32 = 2
} FaissIndicesDataType;

/* faiss::gpu::GpuDistanceParams (faiss/gpu/GpuDistance.h:32-152): the reference's field names, in its order, for the
   fields implemented here (no vectorNorms, ignoreOutDistances, use_cuvs; device is an ordinal, not -1).
   - k in [1, 2048]: k-NN, outDistances / outIndices [numQueries][k].  k = -1: all pairwise distances,
     outDistances [numQueries][numVectors], outIndices unused.  Every distance is the one GpuIndexFlat returns, bit for
     bit (a direct-form sum in dimension order, no ||x||^2 + ||y||^2 - 2<x, y> expansion); for inner product and
     Jaccard the raw similarity; NaN as the CPU computes it.
   - vectorType == queryType is required.  fp16 / bf16 inputs are widened to fp32 exactly on the device.
   - *RowMajor = 0: the input is [dims][num], num innermost.
   - outIndicesType I32 is refused when numVectors > INT32_MAX (the reference narrows silently).
   - Any pointer may be host or device resident.  A host-resident k = -1 matrix is computed in blocks of <= 256 MiB. */
typedef struct FaissGpuDistanceParams {
    FaissMetricType metric;
    float metricArg;
    int k;
    int dims;
    const void* vectors;
    FaissDistanceDataType vectorType;
    int vectorsRowMajor;
    idx_t numVectors;
    const void* queries;
    FaissDistanceDataType queryType;
    int queriesRowMajor;
    idx_t numQueries;
    float* outDistances;
    FaissIndicesDataType outIndicesType;
    void* outIndices;
    int device;
} FaissGpuDistanceParams;
/* faiss::gpu::bfKnn(res, params).  Arguments are validated before any CUDA call: -2 with a message. */
FB200_API int faiss_b200_bfKnn_params(FaissStandardGpuResources* res, const FaissGpuDistanceParams* params);
/* faiss::gpu::bfKnn_tiling (faiss/gpu/GpuDistance.cu:457-570): vectors / queries cut into shards of at most
   vectorsMemoryLimit / queriesMemoryLimit bytes (0: no limit).  The sharded input must be host-resident and row-major,
   k > 0.  The result equals faiss_b200_bfKnn_params's bit for bit. */
FB200_API int faiss_b200_bfKnn_tiling(FaissStandardGpuResources* res, const FaissGpuDistanceParams* params, size_t vectorsMemoryLimit, size_t queriesMemoryLimit);

/* ---- instrumentation (bench.py): kernels launched by this library so far; optional CUDA-event
   timing of a named kernel ("flat_tc") on its launching stream ---- */
FB200_API long long faiss_b200_launch_count(void);
FB200_API void faiss_b200_kernel_timing(int enable);
FB200_API int faiss_b200_kernel_timing_collect(const char* name, double* ms_out, int* launches_out);

/* ---- host-side utilities of the path (no GPU needed) ----
   rand_perm: faiss/utils/random.cpp:188-199; split_clusters: faiss/impl/ClusteringHelpers.cpp:177-240;
   merge_knn_results: faiss/utils/Heap.cpp:166-238 (all_* laid out [nshard][n][k]) */
FB200_API int faiss_b200_rand_perm(int* perm, size_t n, int64_t seed);
FB200_API int faiss_b200_split_clusters(size_t d, size_t k, size_t n, float* hassign, float* centroids, int* nsplit_out);
FB200_API int faiss_b200_merge_knn_results_host(idx_t n, idx_t k, int nshard, FaissMetricType metric, const float* all_distances, const idx_t* all_labels, float* distances, idx_t* labels);

/* ================= tier 2: kernel seams, DEVICE pointers, enqueued on the default stream ======= */
/* role of runL2Norm (faiss/gpu/impl/L2Norm.cu:176) */
FB200_API int b200_l2_norms(FaissStandardGpuResources* res, int device, const float* x, idx_t n, int d, float* norms);
/* role of bfKnnOnDevice (faiss/gpu/impl/Distance.cuh:300), exact SIMT arithmetic */
FB200_API int b200_flat_search_exact(FaissStandardGpuResources* res, int device, const float* Y, idx_t N, int d, const float* Q, idx_t nq, int k, FaissMetricType metric, float* D, idx_t* I);
/* faiss_b200_bfKnn_params for k = -1 into a host-resident matrix, with a block budget of page_bytes instead of 256 MiB */
FB200_API int b200_pairwise_paged(FaissStandardGpuResources* res, const FaissGpuDistanceParams* params, size_t page_bytes);
/* role of merge_knn_results (faiss/utils/Heap.cpp:166-238) on the device: in [nq, nshard, k] */
FB200_API int b200_topk_merge(FaissStandardGpuResources* res, int device, const float* D_in, const idx_t* I_in, idx_t nq, int nshard, int k_in, const idx_t* id_offsets /* device, [nshard] or NULL */, int k, FaissMetricType metric, float* D, idx_t* I);
/* unit-test seam for the tensor-core path: S[nq, roundup(N,256)] = Q16 . Y16^T (fp16 inputs) */
FB200_API int b200_flat_tc_scores_debug(FaissStandardGpuResources* res, int device, const void* Q16, idx_t nq, const void* Y16, idx_t N, int dpad, float* S);
/* the same for int8 rows of 128: S = the exact int32 dot products Q8 . Y8^T, as floats */
FB200_API int b200_flat_tc_scores_debug_s8(FaissStandardGpuResources* res, int device, const void* Q8, idx_t nq, const void* Y8, idx_t N, float* S);
/* role of IVFBase::searchCoarseQuantizer_ (faiss/gpu/impl/IVFBase.cu:509-545): nprobe nearest centroids per query */
FB200_API int b200_ivf_coarse(FaissStandardGpuResources* res, int device, const float* centroids, idx_t nlist, int d, const float* Q, idx_t nq, int nprobe, FaissMetricType metric, float* coarse_dis, idx_t* coarse_ids);
/* role of Clustering's index.search(n, x, 1) (faiss/Clustering.cpp:270-290): nearest centroid of every point */
FB200_API int b200_kmeans_assign(FaissStandardGpuResources* res, int device, const float* centroids, idx_t k, int d, const float* x, idx_t n, FaissMetricType metric, float* dis, idx_t* assign);
/* role of runIVFInterleavedScan (faiss/gpu/impl/IVFInterleaved.cu:179): lists are row-major fp32 runs of one arena,
   list l = elements [list_start[l], +list_len[l]); probes [nq, nprobe] (-1 = skip) */
FB200_API int b200_ivfflat_scan(FaissStandardGpuResources* res, int device, const float* Q, idx_t nq, int d, const idx_t* probes, int nprobe, const int64_t* list_start, const int* list_len, const float* arena_vecs, const idx_t* arena_ids, idx_t arena_elems, int k, FaissMetricType metric, float* D, idx_t* I);
/* role of runPQScanMultiPassNoPrecomputed + pqCodeDistances (faiss/gpu/impl/PQScanMultiPassNoPrecomputed-inl.cuh:527,
   PQCodeDistances-inl.cuh:591) over vector-major [len][M] codes; pq_centroids [M][256][d/M] */
FB200_API int b200_ivfpq_scan(FaissStandardGpuResources* res, int device, const float* Q, idx_t nq, int d, const idx_t* probes, const float* coarse_dis, int nprobe, const float* coarse_centroids, const float* pq_centroids, int M, const int64_t* list_start, const int* list_len, const uint8_t* arena_codes, const idx_t* arena_ids, int k, FaissMetricType metric, float* D, idx_t* I);
/* role of IVFBase::addVectorsToLists_ + runIVFAppend (faiss/gpu/impl/IVFBase.cu:693-905, IVFAppend.cu:265): append n
   encoded rows to their lists (stable order), list_len advanced on the device; capacity is the caller's business */
FB200_API int b200_ivf_append(FaissStandardGpuResources* res, int device, const uint8_t* rows, const idx_t* ids, const idx_t* assign, idx_t n, int code_size, idx_t nlist, const int64_t* list_start, int* list_len, uint8_t* arena_codes, idx_t* arena_ids);
FB200_API int b200_pq_encode(FaissStandardGpuResources* res, int device, const float* residuals, idx_t n, int d, int M, const float* pq_centroids, uint8_t* codes);
FB200_API int b200_kmeans_update(FaissStandardGpuResources* res, int device, const float* x, const idx_t* assign, idx_t n, int d, idx_t k, float* sums, float* counts, float* centroids);

#ifdef __cplusplus
}
#endif
#endif
