/*
 * snap2lmdb.c — cache-directory interchange between this library's snapshot file and the
 * reference's LMDB store.  TEST INFRASTRUCTURE (SURVEY.md §8 f3): it links the COMPILED REFERENCE
 * (oracle/_ref/libcachemap_ref.so: its filemap_* and the mdb_* of its vendored LMDB fork) and the
 * oracle's LZ4 decoder; nothing of it is part of the product library, which keeps LMDB out.
 *
 *   snap2lmdb to-lmdb   <cachemap_b200.snap> <cachedir> <capacity> <pshift>
 *       every record of the snapshot is decoded to its page and stored with the reference's own
 *       filemap_set (cachemap/filemap.c:112-158) under its original timestamp: <cachedir> then holds
 *       filemap.0..31 exactly as the reference writes them (filemap.c:57,71-72,140-147) and the
 *       reference's cachemap_get serves the pages the GPU path stored.
 *   snap2lmdb from-lmdb <cachedir> <cachemap_b200.snap> <pshift>
 *       walks the 32 LMDB environments with a read-only cursor and writes every value (the 24-byte
 *       data_prefix + LZ4 block or raw page) with its attribute (the put timestamp) as one snapshot
 *       record; the GPU library restores such a file on first use (cmb200_load).
 *
 * Snapshot format: edge_fuse_b200/csrc/engine.cu ("CMB200S1"), restated in oracle/snapshot.py.
 * The LMDB prototypes below are declarations of the fork's public interface (cachemap/lmdb.h:
 * 242-260, 288-330, 374-400, 1320) written out here because the header is not shipped with the repo.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

/* ---- the reference's public API (include/filemap.h mirrors cachemap/filemap.h) ---- */
#include "filemap.h"

/* ---- LMDB (fork with node attributes) ---- */
typedef struct MDB_env MDB_env;
typedef struct MDB_txn MDB_txn;
typedef struct MDB_cursor MDB_cursor;
typedef unsigned int MDB_dbi;
typedef struct MDB_val { size_t mv_size; void *mv_data; } MDB_val;
#define MDB_NOSUBDIR 0x4000
#define MDB_RDONLY 0x20000
#define MDB_NOTLS 0x200000
#define MDB_INTEGERKEY 0x08
#define MDB_FIRST 0
#define MDB_NEXT 8
int mdb_env_create(MDB_env **env);
int mdb_env_set_maxreaders(MDB_env *env, unsigned int readers);
int mdb_env_open(MDB_env *env, const char *path, unsigned int flags, unsigned int mode);
void mdb_env_close(MDB_env *env);
int mdb_txn_begin(MDB_env *env, MDB_txn *parent, unsigned int flags, MDB_txn **txn);
void mdb_txn_abort(MDB_txn *txn);
int mdb_dbi_open(MDB_txn *txn, const char *name, unsigned int flags, MDB_dbi *dbi);
int mdb_cursor_open(MDB_txn *txn, MDB_dbi dbi, MDB_cursor **cursor);
void mdb_cursor_close(MDB_cursor *cursor);
int mdb_cursor_get(MDB_cursor *cursor, MDB_val *key, MDB_val *data, int op);
int mdb_get_attr(MDB_txn *txn, MDB_dbi dbi, MDB_val *key, MDB_val *data, uint64_t *attrp);

/* ---- oracle ---- */
int ef_lz4_decode(const uint8_t *src, int src_cap, uint8_t *dst, int n);

struct snap_header { char magic[8]; uint32_t version, pshift; uint64_t records, bytes; uint32_t flags, pad[7]; };
struct snap_record { uint64_t ts, fp_hi, fp_lo; uint32_t len, zero; };

static int
to_lmdb(const char *snap, char *dir, uint64_t capacity, int pshift)
{
	FILE *f = fopen(snap, "rb");
	struct snap_header h;
	if (f && fread(&h, sizeof(h), 1, f) == 1 && memcmp(h.magic, "CMB200E1", 8) == 0) {
		/* a sealed base (cmb200_set_file_key): its records are ciphertext, and this tool holds no key */
		fprintf(stderr, "snap2lmdb: %s is an encrypted snapshot (CMB200E1): this tool holds no key; open the "
		    "cache directory with the library and its CMB200_KEY_FILE, and write it without a key first\n", snap);
		fclose(f);
		return 1;
	}
	if (f) rewind(f);
	if (!f || fread(&h, sizeof(h), 1, f) != 1 || memcmp(h.magic, "CMB200S1", 8) != 0 || (int)h.pshift != pshift) {
		fprintf(stderr, "snap2lmdb: %s is not a snapshot with pshift %d\n", snap, pshift);
		return 1;
	}
	/* a base whose chain has deltas next to it is not the whole store (bytes 40..47: the chain id) */
	uint64_t chain;
	char d1[4096];
	memcpy(&chain, &h.pad[1], 8);
	snprintf(d1, sizeof(d1), "%s.d1", snap);
	if (chain != 0 && access(d1, R_OK) == 0) {
		fprintf(stderr, "snap2lmdb: %s has deltas next to it (%s ...): fold the chain first: open the cache "
		    "directory with the library, which loads base and deltas, and call cachemap_checkpoint\n", snap, d1);
		return 1;
	}
	const size_t bsize = (size_t)1 << pshift;
	struct filemap *fm = filemap_create(dir, capacity, 12, pshift);
	if (!fm) { fprintf(stderr, "snap2lmdb: filemap_create(%s) failed\n", dir); return 1; }
	uint8_t *rec = malloc(24 + bsize + 2048), *page = malloc(bsize);
	uint64_t done = 0;
	for (; done < h.records; done++) {
		struct snap_record r;
		if (fread(&r, sizeof(r), 1, f) != 1 || r.len < 24 || r.len > 24 + bsize + 1024) break;
		size_t padded = ((size_t)r.len + 15) & ~(size_t)15;
		if (fread(rec, padded, 1, f) != 1) break;
		uint128_t key;
		int32_t clen;
		memcpy(&key, rec, 16);
		memcpy(&clen, rec + 16, 4);
		if (clen == 0) memcpy(page, rec + 24, bsize);
		else if (ef_lz4_decode(rec + 24, clen, page, (int)bsize) != clen) break;
		filemap_set(fm, &key, page, r.ts);              /* recompresses with the reference's LZ4: same bytes */
	}
	fclose(f);
	printf("to-lmdb: %lu of %lu records stored, %lu entries\n", (unsigned long)done, (unsigned long)h.records,
	    (unsigned long)filemap_entries(fm));
	/* no filemap_free: mdb_env_close is enough for durability here (MDB_NOSYNC stores still sit in the page cache /
	 * tmpfs), and the process exits */
	return done == h.records ? 0 : 1;
}

static int
from_lmdb(const char *dir, const char *snap, int pshift)
{
	const size_t bsize = (size_t)1 << pshift;
	FILE *f = fopen(snap, "wb");
	if (!f) return 1;
	struct snap_header h;
	memset(&h, 0, sizeof(h));
	memcpy(h.magic, "CMB200S1", 8);
	h.version = 1; h.pshift = (uint32_t)pshift;
	fwrite(&h, sizeof(h), 1, f);
	static const uint8_t zeros[16];
	for (int i = 0; i < FILEMAP_SHARD_NUM; i++) {
		char path[4096];
		snprintf(path, sizeof(path), "%s/filemap.%d", dir, i);
		MDB_env *env = NULL; MDB_txn *txn = NULL; MDB_cursor *cur = NULL; MDB_dbi dbi = 0;
		if (mdb_env_create(&env) || mdb_env_set_maxreaders(env, 32) ||
		    mdb_env_open(env, path, MDB_NOSUBDIR | MDB_RDONLY | MDB_NOTLS, 0664) ||
		    mdb_txn_begin(env, NULL, MDB_RDONLY, &txn) || mdb_dbi_open(txn, NULL, MDB_INTEGERKEY, &dbi) ||   /* filemap.c:80 */
		    mdb_cursor_open(txn, dbi, &cur)) {
			fprintf(stderr, "snap2lmdb: cannot read %s\n", path);
			return 1;
		}
		MDB_val k, v;
		for (int rc = mdb_cursor_get(cur, &k, &v, MDB_FIRST); rc == 0; rc = mdb_cursor_get(cur, &k, &v, MDB_NEXT)) {
			uint64_t key, ts = 0;
			memcpy(&key, k.mv_data, 8);
			MDB_val kk = { sizeof(key), &key }, vv;
			if (mdb_get_attr(txn, dbi, &kk, &vv, &ts) != 0 || vv.mv_size < 24 || vv.mv_size > 24 + bsize + 1024) {
				fprintf(stderr, "snap2lmdb: odd record in %s\n", path);
				return 1;
			}
			struct snap_record r = { ts, 0, 0, (uint32_t)vv.mv_size, 0 };
			size_t padn = (16 - (vv.mv_size & 15)) & 15;
			fwrite(&r, sizeof(r), 1, f);
			fwrite(vv.mv_data, vv.mv_size, 1, f);
			if (padn) fwrite(zeros, padn, 1, f);
			h.records++;
			h.bytes += vv.mv_size;
		}
		mdb_cursor_close(cur);
		mdb_txn_abort(txn);
		mdb_env_close(env);
	}
	fseek(f, 0, SEEK_SET);
	fwrite(&h, sizeof(h), 1, f);
	fclose(f);
	printf("from-lmdb: %lu records\n", (unsigned long)h.records);
	return 0;
}

int
main(int argc, char **argv)
{
	if (argc == 6 && strcmp(argv[1], "to-lmdb") == 0)
		return to_lmdb(argv[2], argv[3], strtoull(argv[4], NULL, 0), atoi(argv[5]));
	if (argc == 5 && strcmp(argv[1], "from-lmdb") == 0)
		return from_lmdb(argv[2], argv[3], atoi(argv[4]));
	fprintf(stderr, "usage: snap2lmdb to-lmdb <snap> <cachedir> <capacity> <pshift>\n"
	    "       snap2lmdb from-lmdb <cachedir> <snap> <pshift>\n");
	return 2;
}
