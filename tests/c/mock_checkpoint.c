/* The CPU stand-in engine (mock_engine.c) with a snapshot call that takes its time, TEST
 * INFRASTRUCTURE ONLY (tests/test_checkpoint_logic.py).  cmb200_save_set writes no file: it sleeps
 * MOCK_SAVE_US and counts its calls, so that a driver can see when the drop-in's CMB200_CHECKPOINT_SEC
 * saves run and whether the callers of cachemap_put wait for them.  cmb200_load_set finds nothing to
 * load.  Nothing of the product links against this file. */
#include "mock_engine.c"

#define MOCK_SAVE_US 1000000

static int saves_started, saves_done;

int cmb200_save_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	(void)engines; (void)g; (void)path;
	__atomic_fetch_add(&saves_started, 1, __ATOMIC_SEQ_CST);
	usleep(MOCK_SAVE_US);
	__atomic_fetch_add(&saves_done, 1, __ATOMIC_SEQ_CST);
	if (records_out) *records_out = 0;
	return 0;
}
int cmb200_load_set(cmb200_engine *const *engines, int g, const char *path, uint64_t *records_out) {
	(void)engines; (void)g; (void)path; if (records_out) *records_out = 0;
	snprintf(err_buf, sizeof(err_buf), "mock: no snapshot files"); return -1;
}

/* saves begun and saves ended so far */
void mock_save_counts(int *started, int *done) {
	*started = __atomic_load_n(&saves_started, __ATOMIC_SEQ_CST);
	*done = __atomic_load_n(&saves_done, __ATOMIC_SEQ_CST);
}
