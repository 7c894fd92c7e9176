/*
 * mlease_host.h -- C entry points of the host job layer (libmlease_host.so; ml-ease_b200/host/).
 * The reference's job classes (the com/linkedin/mlease/regression/jobs/ sources) keep their names, config keys (java
 * .properties job file, com/linkedin/mapred/JobConfig.java:78-90), avro schemas (the .avsc files under src/main/avro/) and output
 * directory layout; the arithmetic goes through include/mlease_b200.h.  CLI: `mlease_regression <job class> <config>`
 * mirrors `hadoop jar … com.linkedin.mlease.regression.jobs.Regression <config>` (jobs/Regression.java:88-98).
 */
#ifndef MLEASE_HOST_H
#define MLEASE_HOST_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
/* job_class: Regression | RegressionPrepare | RegressionAdmmTrain | RegressionTest | RegressionTestLoglik |
 * RegressionNaiveTrain | ItemModelTest | ItemModelTestLoglik | ItemModelTrain | ItemModelGridTest (README aliases
 * AdmmPrepare/AdmmTrain/AdmmTest/AdmmTestLoglik/NaiveTrain accepted).  ItemModelGridTest is not a reference job: it scores held-out
 * records with every (intercept lambda, default lambda) model ItemModelTrain wrote for their key, writes pred (and predVar, the
 * predictive variance under the diagonal posterior, with compute.var) per grid point under output.base.path/lambda-<il>_<dl>/, and
 * one test log-likelihood per grid point under output.base.path/_loglik/.
 * Returns 0, or non-zero with the message (the reference's IOException / RuntimeException text) in mlease_job_last_error(). */
int mlease_job_run(const char* job_class, const char* config_path);
const char* mlease_job_last_error(void);

/* Deterministic branches of RegressionPrepare (jobs/RegressionPrepare.java:154-186): per-record partition keys (positives
 * replicated onto consecutive partitions mod nblocks when the key is drawn at random) and the prepared float weight. */
int mlease_prepare_keys(int64_t nrows, const int32_t* base_key, const int32_t* response, const double* weight_in, int32_t nblocks,
                        int32_t num_click_replicates, int32_t random_key_mode, int32_t* out_keys, int32_t* out_nkeys, float* out_weight);
/* PartitionIdAssigner ids (sorted Utf8 order of "<lambda>#<key>", jobs/PartitionIdAssigner.java:79-88) and NaivePartitioner
 * partitions (id % R, else abs(String.hashCode()) % R, jobs/RegressionNaiveTrain.java:269-283). keys: NUL-separated. */
int mlease_partition_ids(int32_t nkeys, const char* keys_packed, const float* lambdas, int32_t L, int32_t num_reducers, int32_t* out_ids,
                         int32_t* out_partition, int32_t* out_hash_partition);
/* Java Float.toString (model keys "1.0", "1.0#3"). */
int mlease_java_float_to_string(float f, char* buf, int32_t buflen);
/* Worker threads of the host layer (block-parallel avro decode / encode / deflate): n > 0 sets the count (at most 64), 0 returns to
 * the default (MLEASE_HOST_THREADS, else the CPUs this process may run on).  Returns the count in effect. */
int mlease_host_set_threads(int32_t n);
/* Record ingest of the job layer as a library call: prepared records (raw = 0: a file or a directory of RegressionPrepareOutput
 * files, jobs/RegressionAdmmTrain.java:677-690 -> llf/LibLinearDataset.java:413-484) or raw records (raw = 1: one file, the
 * RegressionTest input) into CSR arrays with global feature ids in first-seen order; feature k is "name" or "name\u0001term"
 * (llf/LibLinearDataset.java:456-479).  Blocks of the container files are decoded on all host threads (MLEASE_HOST_THREADS);
 * generic != 0 forces the sequential generic decoder (same result; the tests compare the two). */
typedef struct mlease_rows mlease_rows;
int mlease_rows_read(const char* path, int32_t raw, int32_t binary_feature, int32_t generic, mlease_rows** out);
int64_t mlease_rows_count(const mlease_rows* r, int64_t* nnz, int32_t* nfeatures);   /* returns the number of records */
int mlease_rows_get(const mlease_rows* r, int64_t* rowptr, int32_t* colidx, float* vals, int32_t* response, float* weight, float* offset);
const char* mlease_rows_feature(const mlease_rows* r, int32_t k);
const char* mlease_rows_key(const mlease_rows* r, int64_t i);
void mlease_rows_free(mlease_rows* r);
/* Model files as the jobs write them (LinearModelAvro {key, model}; with uplusx != NULL RegressionTrainOutput {key, model, uplusx},
 * jobs/RegressionAdmmTrain.java:706-711; intercept first, models/LinearModel.java:697-720).  names / keys: NUL-separated lists;
 * coefs, uplusx: [nmodels][nfeatures + 1], intercept last.  generic != 0 selects the Value-tree encoder (tests). */
int mlease_models_write(const char* path, int32_t nfeatures, const char* names, int32_t nmodels, const char* keys, const float* coefs, const float* uplusx,
                        int32_t generic);
/* RegressionTest's output step (jobs/RegressionTest.java:198-236): the records of in_path with every union collapsed to its first
 * non-null branch (utils/Util.java:377-417), record name AdmmTestOutput, and a float field `pred` appended (pred[i] = i-th record). */
int mlease_test_output_write(const char* in_path, const char* out_path, const float* pred, int64_t npred, int32_t generic);
/* RegressionTestLoglik's input step (jobs/RegressionTestLoglik.java:124-151): (response, pred, weight) of the scored records of one
 * file, weight 1 where absent; fills at most `cap` entries, returns the number of records (-1 on error). */
int64_t mlease_scored_read(const char* path, int64_t cap, int32_t* response, float* pred, float* weight, int32_t generic);
/* Avro container round trip (decode every record generically, re-encode with `codec` = "null" | "deflate"). */
int mlease_avro_copy(const char* in_path, const char* out_path, const char* codec, int64_t* nrecords, int64_t* nblocks);
#ifdef __cplusplus
}
#endif
#endif
