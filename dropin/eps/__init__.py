"""Drop-in `eps` package (cppn.py:28-29 `from eps.progress_bar import ...`, `from eps.data_load import ...`). The original project
imports it but does not ship it; these modules map its names onto aphantasia_b200."""
