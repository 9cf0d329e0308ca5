/* Interface compatibility header: the class / function / constant names, signatures and values declared here are those of
 * gr-rfid's installed public header of the same name (nkargas/Gen2-UHF-RFID-Reader, Copyright 2014 Nikos Kargas
 * <nkargas@isc.tuc.gr>, GNU General Public License version 3 or later), because blocks built against it must be
 * drop-in replacements.  The implementation behind the interface is this repository's own.  This file is distributed
 * under the GNU General Public License, version 3 or (at your option) any later version; see LICENSE. */
/* rfid/api.h -- symbol visibility for the gr::rfid block library (H100 host blocks).
 * Same macro name the reference installs (gr-rfid/include/rfid/api.h:27-31) so that
 * application code including <rfid/...> compiles unchanged. */
#ifndef INCLUDED_RFID_API_H
#define INCLUDED_RFID_API_H

#include <gnuradio/attributes.h>

#if defined(gnuradio_rfid_EXPORTS)
#define RFID_API __GR_ATTR_EXPORT
#else
#define RFID_API __GR_ATTR_IMPORT
#endif

#endif /* INCLUDED_RFID_API_H */
